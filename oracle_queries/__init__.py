"""The ray-query oracle (test infrastructure): oracle_queries/queries.cpp + pyqueries.py."""
