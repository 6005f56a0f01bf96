from .epipolar_sampler import EpipolarSampler, EpipolarSampling
from .epipolar_transformer import EpipolarTransformer, EpipolarTransformerCfg, ImageSelfAttentionWrapper
from .image_self_attention import ImageSelfAttention, ImageSelfAttentionCfg
from .positional_encoding import PositionalEncoding
from .transformer import Attention, FeedForward, PreNorm, Transformer
from .depth_predictor_monocular import DepthPredictorMonocular
from .encoder_tail import EncoderEpipolarTail, EncoderTailCfg
from .gaussian_adapter import GaussianAdapter, GaussianAdapterCfg
from .backbone import BackboneDino, BackboneDinoCfg, BackboneResnet, BackboneResnetCfg, get_backbone
from .encoder_epipolar import EncoderEpipolar, EncoderEpipolarCfg
