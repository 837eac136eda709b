"""The sample-variance oracle (test infrastructure): oracle_variance/variance.cpp + pyvariance.py."""
