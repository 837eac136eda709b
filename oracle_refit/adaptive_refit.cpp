/* The Adaptive-sampler oracle (oracle_adaptive/adaptive.cpp, included whole and unchanged) with orc_scene_refit_mesh (refit.h) —
 * TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into oracle/_build/liboracle_adaptive_refit.so and loaded by
 * oracle_refit/pyrefit.py (AdaptiveRefitOracleScene), so that Adaptive per-pixel counts can be checked on a refit mesh. */
#include "../oracle_adaptive/adaptive.cpp"
#include "refit.h"
