// Path-compatible with cupoch/geometry/rgbdimage.h: see cupoch/cupoch_b200_facade.h.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
