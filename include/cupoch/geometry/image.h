// Path-compatible with cupoch/geometry/image.h: geometry::Image as a holder of pixels (no filters, pyramids or IO).
// See cupoch/cupoch_b200_facade.h.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
