"""H100-native drop-in for the checkpoint-snapshot path of NVIDIA Resiliency Extension (NVRx).

Only ``nvidia_resiliency_ext.checkpointing`` is provided (see DESIGN.md for the scope): the import paths,
class names and call signatures mirror the reference so NeMo / PyTorch-Lightning / Megatron callers are
unchanged, while the snapshot itself runs in ``libnvrx_snap.so`` (hand-written sm_90a kernels).
"""

__version__ = "0.1.0+b200"
