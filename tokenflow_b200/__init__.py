"""tokenflow_b200 — H100-native (sm_90a) implementation of TokenFlow's per-denoise-step hot path.

Layout (only what the path needs):
    csrc/               CUDA kernels + the C-ABI (include/tokenflow_b200.h)
    ops.py              ctypes binding; `CudaOps` = one kernel launch per operator, no fallback
    tokenflow_utils.py  drop-in for the reference hook layer (same names / signatures)
    util.py             drop-in for the names the drivers import from `util`
    sd_unet.py, scheduler.py   diffusers-shaped random-init SD UNet + DDIM (diffusers is not installed)
    editor.py           the caller: the reference `batched_denoise_step` loop as one CUDA-graphed fused step, 1..N GPUs
    preprocess.py       the stage in front: DDIM inversion / reconstruction in latent space + the on-disk hand-off
"""
__version__ = "0.2.0"
