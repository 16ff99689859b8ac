// Path-compatible with cupoch/collision/primitives.h: collision::Primitive, Box, Sphere, Capsule, Cylinder, PrimitiveArray on the GPU engine.
// See cupoch/cupoch_b200_facade.h.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
