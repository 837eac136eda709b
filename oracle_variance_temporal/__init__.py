"""The variance temporal denoise oracle (test infrastructure): oracle_variance_temporal/variance_temporal.cpp + pyvariancetemporal.py."""
