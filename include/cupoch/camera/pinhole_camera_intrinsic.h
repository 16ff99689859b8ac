// Path-compatible with cupoch/camera/pinhole_camera_intrinsic.h: camera::PinholeCameraIntrinsic as plain data.
// See cupoch/cupoch_b200_facade.h.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
