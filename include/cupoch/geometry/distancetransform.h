// Path-compatible with cupoch/geometry/distancetransform.h: geometry::DistanceVoxel, geometry::DistanceTransform on the
// GPU engine.  See cupoch/cupoch_b200_facade.h.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
