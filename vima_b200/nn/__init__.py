"""`vima.nn` surface (reference: /root/reference/vima/nn/__init__.py:1-6) on sm_90a kernels."""
from .action import (
    ActionDecoder,
    ActionEmbedding,
    ActionSampler,
    Categorical,
    CategoricalNet,
    ContinuousActionEmbedding,
    MultiCategorical,
    MultiCategoricalNet,
)
from .basic import Conv1D, Embedding, Linear, MLPSequential, build_mlp
from .obj_encoder import (GatoMultiViewRGBEncoder, GatoViTEncoder, MultiViewRGBEncoder, MultiViewRGBPerceiverEncoder, ObjEncoder, ViTEncoder, ViTEncoderRectangular,
                          VisionTransformer)
from .perceiver import ObjectsPerceiverEncoder
from .t5_encoder import T5PromptEncoder, WordEmbedding
from .xattn_gpt import HFGPT, DecodeCache, SlotDecodeCache, SwappedEpisode, XAttnGPT
