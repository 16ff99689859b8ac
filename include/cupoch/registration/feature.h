// Path-compatible with the reference header cupoch/registration/feature.h (Feature, ComputeFPFHFeature,
// ComputeSHOTFeature); the declarations live in the single facade header.
#pragma once
#include "cupoch/cupoch_b200_facade.h"
