"""The denoiser oracle (test infrastructure): oracle_denoise/denoise.cpp + pydenoise.py."""
