"""`import video_transformer` of the reference (model_trainer.py:18, visualize_attention.py) -> this package's models."""
from videotransformer_pytorch_b200.maskfeat import MaskFeat  # noqa: F401
from videotransformer_pytorch_b200.video_transformer import TimeSformer, ViViT, get_vit_base_patch16_224  # noqa: F401
