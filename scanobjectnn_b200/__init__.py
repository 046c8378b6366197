"""scanobjectnn_b200 -- H100-native point-set-abstraction hot path (FPS, ball query / kNN, group,
grouped shared MLP + max-pool, three-NN interpolation) behind the reference's own op names.

Only what the hot path needs lives here: ``csrc/`` (hand-written sm_90a CUDA + the C ABI declared
in include/psa.h) and the host-side mirror of the reference's Python op / layer interface.
"""
__version__ = "0.1.0"
