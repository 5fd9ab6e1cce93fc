"""Example problem definitions (mirrors of test/examples/* of the reference) for the GPU path."""
