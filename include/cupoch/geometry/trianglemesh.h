// Path-compatible with cupoch/geometry/trianglemesh.h: geometry::TriangleMesh (and its MeshBase) with its attributes,
// the two normal computations, the edge list, the four vertex filters, the surface area, uniform sampling, the bounds,
// the cleanup operations, GetSelfIntersectingTriangles and + / += (no IO or primitives).  See cupoch/cupoch_b200_facade.h.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
