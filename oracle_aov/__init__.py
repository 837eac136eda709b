"""The AOV oracle (test infrastructure): oracle_aov/aov.cpp + pyaov.py."""
