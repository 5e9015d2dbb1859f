"""phenaki-pytorch hot path, H100-native (sm_90a).  Drop-in names of the reference package
(/root/reference/phenaki_pytorch/__init__.py:1-4) for the C-ViViT encode + MaskGIT sampling path."""
from .cvivit import CViViT
from .modules import invalidate_weights
from .phenaki import MaskGit, Phenaki, SelfCritic, TokenCritic, make_video

__all__ = ["CViViT", "MaskGit", "TokenCritic", "SelfCritic", "Phenaki", "make_video", "invalidate_weights"]
