"""The mesh-refit oracle (test infrastructure): oracle_refit/refit.cpp + pyrefit.py."""
