"""Shared test tables and scripts (not test modules)."""
