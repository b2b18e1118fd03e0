"""closerlook3d_b200 -- H100-native (Hopper, sm_90a) local-aggregation engine, drop-in for the hot path of
zeliu98/CloserLook3D (see DESIGN.md).  Public surface mirrors the reference:

    closerlook3d_b200.local_aggregation_operators   LocalAggregation, PosPool, AdaptiveWeight, PointWiseMLP, PseudoGrid
    closerlook3d_b200.pt_utils                      MaskedQueryAndGroup, MaskedMaxPool, MaskedUpsample, ...
    closerlook3d_b200.ext                           the five `_ext` functions
    closerlook3d_b200.shim.install()                run the reference's own models/ on this package
    closerlook3d_b200.graphed.GraphedStep           CUDA-graph replay of a training step
    closerlook3d_b200.dist                          batch sharding + gradient all-reduce

The native library (closerlook3d_b200/libcl3d.so, C ABI in include/cl3d.h) is built in-tree by
`python -m closerlook3d_b200.build`; nothing here falls back to CPU or to PyTorch kernels when it is missing.
"""
__version__ = "0.1.0"
