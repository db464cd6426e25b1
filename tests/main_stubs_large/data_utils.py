"""Stub of the reference's ``data_utils`` (Main.py:13 star-imports it; nothing of it is called directly)."""
