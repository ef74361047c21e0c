"""Drop-in mirror of the reference's ``nets`` package for the graph-attention hot path."""
from . import (dp_attention_transformer, dp_attention_transformer_oc20, equiformer_md17_dens,  # noqa: F401
               graph_attention_transformer, graph_attention_transformer_md17,
               graph_attention_transformer_oc20)                                                          # (register models)
from .registry import list_models, model_entrypoint, register_model  # noqa: F401
from .graph_attention_transformer import (  # noqa: F401
    DepthwiseTensorProduct, EdgeDegreeEmbeddingNetwork, FeedForwardNetwork, GraphAttention,
    GraphAttentionTransformer, SeparableFCTP, TransBlock)
from .dp_attention_transformer import (  # noqa: F401
    DotProductAttention, DotProductAttentionTransformer, DotProductAttentionTransformerMD17, DPTransBlock)
from .dp_attention_transformer_oc20 import DotProductAttentionTransformerOC20  # noqa: F401
from .tensor_product_rescale import (  # noqa: F401
    FullyConnectedTensorProductRescale, LinearRS, TensorProductRescale)
