// Path-compatible with cupoch/geometry/voxelgrid.h: geometry::Voxel, geometry::VoxelGrid (creation from a point cloud or
// a triangle mesh, CreateDense, CreateFromOccupancyGrid, CheckIfIncluded, carving, += / AddVoxels, painting,
// SelectByIndex) on the GPU engine.  See cupoch/cupoch_b200_facade.h.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
