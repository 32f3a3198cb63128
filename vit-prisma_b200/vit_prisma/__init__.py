"""vit_prisma -- H100-native drop-in for the two hot paths of Prisma-Multimodal/ViT-Prisma.

Same import paths as the reference package (``vit_prisma.models.base_vit.HookedViT``,
``vit_prisma.prisma_tools.hook_point.HookPoint``, ``vit_prisma.sae...``); the arithmetic lives in
``lib/libprisma_b200.so`` (hand-written sm_90a CUDA, C ABI in ``include/prisma_b200.h``).
"""
__version__ = "0.1.0"
