// Path-compatible with cupoch/collision/collision.h: collision::CollisionResult, collision::ComputeIntersection on the GPU engine.
// See cupoch/cupoch_b200_facade.h.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
