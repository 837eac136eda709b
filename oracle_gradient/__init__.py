"""The temporal gradient oracle (test infrastructure): oracle_gradient/gradient.cpp + pygradient.py."""
