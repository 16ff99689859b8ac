// Path-compatible with cupoch/geometry/trianglemesh.h: geometry::TriangleMesh with its attributes and the two normal
// computations (no filtering, sampling or IO).  See cupoch/cupoch_b200_facade.h.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
