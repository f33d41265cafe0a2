"""instancediffusion_b200 -- H100-native (sm_90a) kernels + drop-in host mirror for the
InstanceDiffusion sampling hot path (SURVEY.md section 8)."""

__version__ = "0.1.0"


def set_storage_dtype(dtype):
    """Select the 16-bit storage type of activations / packed weights (torch.float16, the default and the
    reference's autocast type, or torch.bfloat16 -> libidiff_b200_bf16.so).  See ops.set_storage_dtype."""
    from . import ops
    ops.set_storage_dtype(dtype)
