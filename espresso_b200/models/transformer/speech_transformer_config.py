"""Model configuration with the reference's field names
(espresso/models/transformer/speech_transformer_config.py:20-300; YAML recipes under
examples/asr_librispeech/config/)."""
import ast
from dataclasses import dataclass, field
from typing import Optional

DEFAULT_MAX_SOURCE_POSITIONS = 10240


@dataclass
class SpeechEncDecBaseConfig:
    embed_dim: int = 512
    ffn_embed_dim: int = 2048
    layers: int = 6
    attention_heads: int = 8
    normalize_before: bool = True
    learned_pos: bool = False
    relative_positional_embeddings: bool = False
    share_learned_relative_positional_embeddings_across_layers: bool = False
    share_learned_relative_positional_embeddings_across_heads: bool = False
    layerdrop: float = 0.0


@dataclass
class SpeechEncoderConfig(SpeechEncDecBaseConfig):
    conv_channels: Optional[str] = "[64, 64, 128, 128]"
    conv_kernel_sizes: Optional[str] = "[(3, 3), (3, 3), (3, 3), (3, 3)]"
    conv_strides: Optional[str] = "[(1, 1), (2, 2), (1, 1), (2, 2)]"
    layer_type: str = "transformer"  # "transformer" | "conformer"
    depthwise_conv_kernel_size: int = 31
    transformer_context: Optional[str] = None
    chunk_size: int = 0  # > 0: chunk-streaming self-attention (speech_transformer_config.py:85-100)
    chunk_left_window: int = 0
    chunk_right_window: int = 0


@dataclass
class SpeechDecoderConfig(SpeechEncDecBaseConfig):
    input_dim: int = 512
    output_dim: int = 512
    # relaxed encoder-decoder attention in training (--decoder-relaxed-attention-weight; fairseq/modules/
    # multihead_attention.py:869-872): probabilities (1 - w) p + w / src_len; 0 disables it
    relaxed_attention_weight: float = 0.0


@dataclass
class SpeechTransformerConfig:
    activation_fn: str = "relu"
    dropout: float = 0.2
    attention_dropout: float = 0.2
    activation_dropout: float = 0.2
    encoder: SpeechEncoderConfig = field(default_factory=SpeechEncoderConfig)
    decoder: SpeechDecoderConfig = field(default_factory=SpeechDecoderConfig)
    share_decoder_input_output_embed: bool = False
    # scheduled sampling of the Transformer decoder (espresso/models/transformer/speech_transformer_config.py:260-272):
    # probability of feeding the TRUTH token per epoch from start_scheduled_sampling_epoch on; the last value persists
    scheduled_sampling_probs: tuple = (1.0,)
    start_scheduled_sampling_epoch: int = 1
    no_cross_attention: bool = False
    max_source_positions: Optional[int] = DEFAULT_MAX_SOURCE_POSITIONS
    max_target_positions: Optional[int] = 1024
    layernorm_embedding: bool = False
    no_scale_embedding: bool = False
    no_token_positional_embeddings: bool = False

    @classmethod
    def from_dict(cls, d):
        """Build from a (possibly nested) mapping such as the `model:` section of a recipe YAML."""
        cfg = cls()
        for k, v in d.items():
            if k in ("encoder", "decoder"):
                sub = getattr(cfg, k)
                for ek, ev in v.items():
                    if hasattr(sub, ek):
                        setattr(sub, ek, ev)
            elif hasattr(cfg, k):
                setattr(cfg, k, v)
        return cfg


def eval_str_nested_list_or_tuple(x, type=int):
    """espresso/tools/utils.py `eval_str_nested_list_or_tuple`: "[(3, 3), (3, 3)]" -> nested list."""
    if x is None:
        return None
    if isinstance(x, str):
        x = ast.literal_eval(x)
    return x
