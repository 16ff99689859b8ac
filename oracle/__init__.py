"""The CPU oracle: plain-C restatements of the reference's algorithms, one shared library per restatement.

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__, bench.py's CPU legs and tools/, never by the product
package cupoch_b200/.  build() compiles the libraries, load() opens one, ptr() hands a numpy array to it; the
<name>_py modules wrap each library's functions.
"""
import ctypes
import glob
import hashlib
import json
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
# lib<name>.so is built from <name>.c alone; iss.c and shot.c #include oracle.c to reuse its static helpers
NAMES = ("oracle", "edt", "fps", "iss", "segment_plane", "shot")
# gcc from PATH, not $CC: a build environment's $CC may be a compiler without OpenMP, which would quietly make the
# oracle, and with it bench.py's all-cores CPU baseline, single-threaded
CC = "gcc"
# -ffp-contract=off: every fused multiply-add in the restatements is an explicit fmaf(); -mfma only makes those calls
# inline to hardware FMA (identical results, faster).  No -ffast-math.
CFLAGS = ["-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-Wall", "-Wextra", "-Wno-unused-parameter",
          "-Wno-unused-function", "-Wno-unknown-pragmas"]
# oracle/_build/, or a per-user temporary directory when the tree is read-only
OUT_DIRS = (os.path.join(HERE, "_build"), os.path.join(tempfile.gettempdir(), "cphb_oracle_%d" % os.getuid()))


def _signature():
    """content hash of every oracle source and header, the compiler and the flags: staleness must not depend on file
    mtimes (a copied tree does not keep them), and hashing the whole directory cannot miss an #include"""
    h = hashlib.sha256()
    for path in sorted(glob.glob(os.path.join(HERE, "*.[ch]"))):
        with open(path, "rb") as f:
            h.update(os.path.basename(path).encode() + b"\0" + hashlib.sha256(f.read()).digest())
    h.update(" ".join([CC] + CFLAGS).encode())
    return h.hexdigest()


def _manifest(out):
    try:
        with open(os.path.join(out, "manifest.json")) as f:
            return json.load(f)
    except (OSError, ValueError):
        return {}


def _compile(name, out):
    so = os.path.join(out, "lib%s.so" % name)
    tmp = "%s.%d.tmp" % (so, os.getpid())
    cmd = CFLAGS + ["-shared", "-o", tmp, os.path.join(HERE, name + ".c"), "-lm"]
    # OpenMP only parallelises over points or lines whose results are computed alone: one thread gives the same results
    if subprocess.run([CC, "-fopenmp"] + cmd, capture_output=True).returncode != 0:
        subprocess.check_call([CC] + cmd)
    # a process loading the library concurrently must never open a half-written file
    os.replace(tmp, so)
    return so


def build(name=None, force=False):
    """Build lib<name>.so, or every library when name is None, unless a current one exists -> its path (or a list).

    A library is current when <out>/manifest.json records the signature of today's sources, compiler and flags for
    it.  <out> is oracle/_build/; in a read-only tree a current library there is still used, and otherwise the
    per-user temporary directory takes its place."""
    if name is None:
        return [build(n, force) for n in NAMES]
    sig = _signature()
    tree = OUT_DIRS[0]
    dirs = OUT_DIRS[:1] if os.access(HERE, os.W_OK) or os.access(tree, os.W_OK) else OUT_DIRS
    for out in dirs:
        so = os.path.join(out, "lib%s.so" % name)
        if not force and _manifest(out).get(name) == sig and os.path.exists(so):
            return so
    out = dirs[-1]
    os.makedirs(out, exist_ok=True)
    so = _compile(name, out)
    manifest = _manifest(out)  # read again just before writing: another process may have built another library
    manifest[name] = sig
    tmp = os.path.join(out, "manifest.json.%d.tmp" % os.getpid())
    with open(tmp, "w") as f:
        json.dump(manifest, f, indent=0, sort_keys=True)
    os.replace(tmp, os.path.join(out, "manifest.json"))
    return so


_loaded = {}


def load(name):
    """ctypes.CDLL of lib<name>.so, built first if it is missing or stale; one per process"""
    if name not in _loaded:
        _loaded[name] = ctypes.CDLL(build(name))
    return _loaded[name]


def ptr(a):
    """a contiguous numpy array as a void * argument; None as NULL"""
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)
