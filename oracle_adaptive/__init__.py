"""The Adaptive-sampler oracle (test infrastructure): oracle_adaptive/adaptive.cpp + pyadaptive.py."""
