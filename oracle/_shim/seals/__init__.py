"""Names-only stub (oracle/_shim): the `seals` package the reference's algorithms/mce_irl.py imports."""
