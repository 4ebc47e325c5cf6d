"""coclr_b200 -- sm_90a (H100) kernels + host executor behind the CoCLR pre-training hot path."""
__version__ = "0.1.0"
