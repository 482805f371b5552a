"""Modules mirroring the reference's espnet class surface for the encoder hot path (SURVEY.md 8b)."""
from .attention import RelPositionMultiHeadedAttention
from .conformer_encoder import ConformerEncoder, ConvolutionModule, EncoderLayer
from .ctc import CTC, ProjEncoder
from .embedding import RelPositionalEncoding
from .label_smoothing_loss import LabelSmoothingLoss
from .layer_norm import LayerNorm
from .positionwise_feed_forward import PositionwiseFeedForward
from .repeat import MultiSequential, repeat
from .resnet import Conv1dResNet, Conv3dResNet
from .scorers_ctc import CTCPrefixScorer
from .transformer_decoder import TransformerDecoder

# north_star spelling
Encoder = ConformerEncoder

__all__ = ["ConformerEncoder", "Encoder", "EncoderLayer", "ConvolutionModule", "RelPositionMultiHeadedAttention",
           "PositionwiseFeedForward", "LayerNorm", "RelPositionalEncoding", "MultiSequential", "repeat", "CTC",
           "ProjEncoder", "TransformerDecoder", "CTCPrefixScorer", "LabelSmoothingLoss", "Conv3dResNet", "Conv1dResNet"]
