"""The moment gradient oracle (test infrastructure): oracle_moment_gradient/moment_gradient.cpp + pymomentgradient.py."""
