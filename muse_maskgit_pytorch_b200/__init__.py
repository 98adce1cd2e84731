"""muse_maskgit_pytorch_b200 — Hopper-native (sm_90a) drop-in for the MaskGit.generate() hot path of
lucidrains/muse-maskgit-pytorch.  Same public classes as the reference package (ref: muse_maskgit_pytorch/__init__.py:1-4)
minus the trainer, which is out of scope."""
from .vqgan_vae import VQGanVAE
from .muse_maskgit import Transformer, MaskGit, Muse, MaskGitTransformer, TokenCritic
from .pack_cache import set_pack_cache

__all__ = ["VQGanVAE", "Transformer", "MaskGit", "Muse", "MaskGitTransformer", "TokenCritic", "set_pack_cache"]
