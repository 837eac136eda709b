"""The moment denoiser oracle (test infrastructure): oracle_moments/moments.cpp + pymoments.py."""
