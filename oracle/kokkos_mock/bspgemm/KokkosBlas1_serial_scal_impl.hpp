// Stand-in: SerialScaleInternal lives in KokkosKernels_helpers.hpp of this directory.  TEST INFRASTRUCTURE ONLY.
#pragma once
#include "KokkosKernels_helpers.hpp"
