"""H100-native (sm_90a) forward/backward for the video-transformer hot path of
mx-mark/VideoTransformer-pytorch, behind the reference's own nn.Module surface.

    from videotransformer_pytorch_b200 import TimeSformer, ViViT, MaskFeat

The package is importable without a GPU (module construction, state dicts); any forward needs
libvt_b200.so (python -m videotransformer_pytorch_b200.build) and an H100 (sm_90) — there is no fallback.
"""
from .transformer import (Attention, BasicTransformerBlock, ClassificationHead,  # noqa: F401
                          DividedSpatialAttentionWithPreNorm, DividedTemporalAttentionWithPreNorm, DropPath,
                          FFNWithPreNorm, MultiheadAttentionWithPreNorm, PatchEmbed, TransformerContainer,
                          get_sine_cosine_pos_emb)
from .video_transformer import TimeSformer, ViViT, get_vit_base_patch16_224  # noqa: F401
from .maskfeat import MaskFeat  # noqa: F401
from .mixup import MixedClip, Mixup  # noqa: F401
from .ops import cross_entropy  # noqa: F401
from .metrics import TopKAccuracy  # noqa: F401

__version__ = '0.1.0'
