"""active_learning_b200 -- H100 (sm_90a) acquisition-scoring engine for the per-round query step
of zeyademam/active_learning.

    from active_learning_b200.query_strategies.get_strategy import get_strategy   # drop-in dispatch
    from active_learning_b200.engine import Engine                                  # raw kernels

The compute path is libalq.so (hand-written CUDA behind a C ABI, include/alq.h); PyTorch is the
allocator / stream / process-group provider.  Importing this package never compiles anything and
never touches the GPU; constructing an Engine without libalq.so + an sm_90 GPU (H100) raises.
"""
__version__ = "0.1.0"
