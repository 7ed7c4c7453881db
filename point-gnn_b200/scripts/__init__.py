"""Command-line twins of the reference's data tools (``scripts/``)."""
