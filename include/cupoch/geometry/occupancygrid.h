// Path-compatible with cupoch/geometry/occupancygrid.h: geometry::OccupancyVoxel, geometry::OccupancyGrid on the GPU
// engine.  See cupoch/cupoch_b200_facade.h.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
