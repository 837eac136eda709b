"""The Adaptive AOV oracle (test infrastructure): oracle_adaptive_aov/adaptive_aov.cpp + pyadaptiveaov.py."""
