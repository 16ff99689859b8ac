// Path-compatible with cupoch/integration/scalable_tsdfvolume.h: see cupoch/cupoch_b200_facade.h.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
