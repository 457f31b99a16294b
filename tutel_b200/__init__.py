"""tutel_b200 - a H100-native (sm_90a, NVLink 4) Mixture-of-Experts framework with the capabilities and API of
microsoft/tutel: ``moe.moe_layer`` with top-k gating and dynamic capacity, switchable DP / EP / sharded-expert
parallelism, all-to-all / FFN pipelining, 2DH, a dropless Megablocks path, ragged collectives, ZeRO helpers,
re-shardable checkpoints - built on hand-written wgmma / TMA kernels and in-kernel NVLink peer-to-peer transfers.

    from tutel_b200 import moe, net, system, jit
    # or, to run code written against the reference unchanged:
    import tutel_b200.compat; tutel_b200.compat.install_as_tutel()
"""
__version__ = '0.1.0'

from . import system as system_init  # noqa: F401  (mirrors tutel/__init__.py)
