"""The temporal denoiser oracle (test infrastructure): oracle_temporal/temporal.cpp + pytemporal.py."""
