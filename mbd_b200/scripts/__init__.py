"""Command-line drivers (python -m mbd_b200.scripts.<name>)."""
