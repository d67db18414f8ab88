"""`import transformer` of the reference (model_trainer.py:17, video_transformer.py:8-10) -> this package's modules."""
from videotransformer_pytorch_b200.transformer import *  # noqa: F401,F403
from videotransformer_pytorch_b200.transformer import (Attention, BasicTransformerBlock, ClassificationHead,  # noqa: F401
                                                       DividedSpatialAttentionWithPreNorm,
                                                       DividedTemporalAttentionWithPreNorm, DropPath, FFNWithPreNorm,
                                                       MultiheadAttentionWithPreNorm, PatchEmbed, TransformerContainer,
                                                       get_sine_cosine_pos_emb)
