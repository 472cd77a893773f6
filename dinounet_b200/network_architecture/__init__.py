"""`dinounet.network_architecture`-style module surface of the native Dino U-Net (see modules.py)."""
from .modules import (  # noqa: F401
    DinoUNet, DINOv3EncoderAdapter, FAPM, SqueezeExcitation, DepthwiseSeparableConv, LearnableUpsampleBlock,
    UNetDecoder, DINOv3_Adapter, SpatialPriorModule, InteractionBlockWithCls, Extractor, ConvFFN, DWConv,
    MSDeformAttn, DinoVisionTransformer, SelfAttentionBlock, SelfAttention, LinearKMaskedBias, Mlp, SwiGLUFFN,
    LayerScale, PatchEmbed, RopePositionEmbedding, StackedConvBlocks, ConvDropoutNormReLU, load_dinov3_model,
    make_backbone,
)
