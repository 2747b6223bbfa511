"""compare_gan_b200 — H100 (sm_90a) GAN training-step and FID-evaluation engine behind
google/compare_gan's ModularGAN / arch_ops surface.  Host code is Python; every per-step
computation is a hand-written CUDA kernel reached through the C-ABI in include/cgan_b200.h.
"""
from . import gin_lite as gin  # noqa: F401
