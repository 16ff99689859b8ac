#!/usr/bin/env python3
"""Prints the marching-cubes tables of UniformTSDFVolume::ExtractTriangleMesh (cupoch_b200/csrc/tsdf.cu and
oracle/tsdf_mesh.c carry the SAME text, written out twice on purpose: product and oracle share a specification, not
code).  The tables are derived here from a stated rule, not copied from any classic table:

- Corners and edges (index conventions).  Corner i of the cube at voxel (x, y, z) is the voxel (x, y, z) + CORNER[i];
  its bit in the cube index is set when its tsdf < 0 (inside).  Edge e runs from its origin corner EDGE[e][:3] along
  axis EDGE[e][3] to the next corner.
- Edge table: edge e is crossed iff its two corners' bits differ.
- Triangle table.  On each of the cube's six faces the crossed edges are joined by segments: two crossed edges by one
  segment; on an ambiguous face (four crossed edges: diagonal corners equal, adjacent corners different) each negative
  corner is cut off by the segment joining its two edges, so the negative corners are kept apart.  The rule reads only
  the face's four signs, so the two cubes sharing a face draw the same segments.  A segment is directed along
  g x N, where N is the face's outward normal and g points from the segment's negative side to its positive side
  within the face; the two cubes sharing a face therefore draw it in opposite directions.  Every crossed edge then has
  one segment leaving and one entering, and following them gives closed polygons whose right-hand normal points from
  negative (inside) to positive tsdf.  Polygons are listed by their smallest edge number, each starting there, and
  each is fan-triangulated from a fixed vertex p0: (p0, p1, p2), (p0, p2, p3), ...  p0 is the first vertex, in polygon
  order, none of whose diagonals joins two edges of one face (a diagonal on a face could meet the neighbouring cube's
  diagonal there and put four triangles on one edge); every polygon has one.
- MC_MAX_TRIS is the largest triangle count of any configuration; output buffers are sized from it.

    python tools/gen_mc_tables.py           # the C block, as it appears in both sources
"""
CORNER = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
EDGE = [(0, 0, 0, 0), (1, 0, 0, 1), (0, 1, 0, 0), (0, 0, 0, 1), (0, 0, 1, 0), (1, 0, 1, 1), (0, 1, 1, 0), (0, 0, 1, 1),
        (0, 0, 0, 2), (1, 0, 0, 2), (1, 1, 0, 2), (0, 1, 0, 2)]
BEGIN, END = "/* BEGIN tables printed by tools/gen_mc_tables.py */", "/* END tables printed by tools/gen_mc_tables.py */"


def edge_corners(e):
    """(origin corner, end corner) of edge e"""
    o = EDGE[e][:3]
    t = list(o)
    t[EDGE[e][3]] += 1
    return CORNER.index(tuple(o)), CORNER.index(tuple(t))


def faces():
    """(corner indices, outward normal) of the six faces"""
    out = []
    for a in range(3):
        for s in (0, 1):
            n = [0, 0, 0]
            n[a] = 2 * s - 1
            out.append(([i for i in range(8) if CORNER[i][a] == s], tuple(n)))
    return out


def face_edges(cs):
    return [e for e in range(12) if set(edge_corners(e)) <= set(cs)]


def neg(ci, i):
    return (ci >> i) & 1


def edge_table(ci):
    return sum(1 << e for e in range(12) if neg(ci, edge_corners(e)[0]) != neg(ci, edge_corners(e)[1]))


def _mid(e):
    a, b = edge_corners(e)
    return [(CORNER[a][k] + CORNER[b][k]) / 2 for k in range(3)]


def _sub(a, b):
    return [a[k] - b[k] for k in range(3)]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    return sum(a[k] * b[k] for k in range(3))


def _mean(ps):
    return [sum(p[k] for p in ps) / len(ps) for k in range(3)]


def face_segments(ci, cs, n):
    """the face rule: directed segments (from edge, to edge) on the face with corners cs and outward normal n"""
    es = [e for e in face_edges(cs) if edge_table(ci) >> e & 1]
    if not es:
        return []
    if len(es) == 2:
        pairs = [(es[0], es[1],
                  _sub(_mean([CORNER[c] for c in cs if not neg(ci, c)]), _mean([CORNER[c] for c in cs if neg(ci, c)])))]
    else:  # ambiguous: cut off each negative corner
        centre = _mean([CORNER[c] for c in cs])
        pairs = []
        for c in cs:
            if neg(ci, c):
                a, b = [e for e in es if c in edge_corners(e)]
                pairs.append((a, b, _sub(centre, CORNER[c])))
    out = []
    for a, b, g in pairs:
        s = _dot(_sub(_mid(b), _mid(a)), _cross(g, n))
        assert s != 0
        out.append((a, b) if s > 0 else (b, a))
    return out


def polygons(ci):
    """the closed, oriented polygons of configuration ci, each starting at its smallest edge, by that edge"""
    nxt = {}
    for cs, n in faces():
        for a, b in face_segments(ci, cs, n):
            assert a not in nxt
            nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values()) == [e for e in range(12) if edge_table(ci) >> e & 1]
    seen, polys = set(), []
    for e in sorted(nxt):
        if e in seen:
            continue
        p = [e]
        while nxt[p[-1]] != e:
            p.append(nxt[p[-1]])
        seen.update(p)
        polys.append(p)
    for p in polys:  # self-check: the Newell normal points from the negative corners to the positive ones
        nrm = [0.0, 0.0, 0.0]
        for i in range(len(p)):
            nrm = [nrm[k] + c for k, c in enumerate(_cross(_mid(p[i]), _mid(p[(i + 1) % len(p)])))]
        grad = [0.0, 0.0, 0.0]
        for e in p:
            a, b = edge_corners(e)
            d = _sub(CORNER[b], CORNER[a]) if neg(ci, a) else _sub(CORNER[a], CORNER[b])
            grad = [grad[k] + d[k] for k in range(3)]
        assert _dot(nrm, grad) > 0, (ci, p)
    return polys


def _on_one_face(e, f):
    return any(set(edge_corners(e)) | set(edge_corners(f)) <= set(cs) for cs, _ in faces())


def fan_start(p):
    """the first vertex of polygon p none of whose fan diagonals lies on a face"""
    return next(s for s in range(len(p)) if not any(_on_one_face(p[s], p[(s + j) % len(p)]) for j in range(2, len(p) - 1)))


def triangles(ci):
    out = []
    for p in polygons(ci):
        s = fan_start(p)
        q = p[s:] + p[:s]
        out += [(q[0], q[k], q[k + 1]) for k in range(1, len(q) - 1)]
    return out


def max_tris():
    return max(len(triangles(ci)) for ci in range(256))


def c_block():
    m = max_tris()
    L = [BEGIN, "#define MC_MAX_TRIS %d /* the most triangles any configuration produces */" % m,
         "/* corner i of a cube: its voxel offset */",
         "MC_TABLE int8_t mc_corner[8][3] = {%s};" % ", ".join("{%d, %d, %d}" % c for c in CORNER),
         "/* edge e: origin corner offset and axis */",
         "MC_TABLE int8_t mc_edge[12][4] = {%s};" % ", ".join("{%d, %d, %d, %d}" % e for e in EDGE),
         "/* bit e: edge e is crossed */", "MC_TABLE uint16_t mc_edge_table[256] = {"]
    for r in range(0, 256, 16):
        L.append("    " + " ".join("0x%03x," % edge_table(ci) for ci in range(r, r + 16)))
    L += ["};", "MC_TABLE uint8_t mc_tri_count[256] = {"]
    for r in range(0, 256, 32):
        L.append("    " + " ".join("%d," % len(triangles(ci)) for ci in range(r, r + 32)))
    L += ["};", "/* the edges of each triangle, -1 past mc_tri_count */", "MC_TABLE int8_t mc_tri_table[256][3 * MC_MAX_TRIS] = {"]
    for ci in range(256):
        t = [e for tri in triangles(ci) for e in tri]
        t += [-1] * (3 * m - len(t))
        L.append("    {%s}," % ", ".join(str(e) for e in t))
    L += ["};", END]
    return "\n".join(L) + "\n"


if __name__ == "__main__":
    print(c_block(), end="")
