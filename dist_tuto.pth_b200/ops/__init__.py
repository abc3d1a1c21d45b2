"""Hand-written sm_90a kernels and their Python entry points (see csrc/)."""
