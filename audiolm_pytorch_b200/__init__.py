"""CUDA-native AudioLM hot path for the H100 (SoundStream codec convs + RVQ, Semantic/Coarse/Fine transformers).

Same class names, constructor kwargs, forward()/generate()/tokenize() signatures and state_dict keys
as lucidrains/audiolm-pytorch (audiolm_pytorch/__init__.py exports the same public names); the arithmetic
underneath is hand-written sm_90a CUDA reached through the C ABI in include/alm_b200.h (libalm_b200.so).
"""
__version__ = "0.2.0"

from .audiolm import (AudioLM, CoarseTransformer, CoarseTransformerWrapper, FineTransformer,  # noqa: E402,F401
                      FineTransformerWrapper, SemanticTransformer, SemanticTransformerWrapper)
from .encodec import EncodecWrapper  # noqa: E402,F401
from .hubert import HubertWithKmeans  # noqa: E402,F401
from .parallel import FlatGradBucket  # noqa: E402,F401
from .soundstream import AudioLMSoundStream, MusicLMSoundStream, SoundStream  # noqa: E402,F401
from .transformer import Transformer  # noqa: E402,F401
from .vq_wav2vec import FairseqVQWav2Vec  # noqa: E402,F401

__all__ = ["AudioLM", "SemanticTransformer", "CoarseTransformer", "FineTransformer", "SemanticTransformerWrapper",
           "CoarseTransformerWrapper", "FineTransformerWrapper", "SoundStream", "AudioLMSoundStream",
           "MusicLMSoundStream", "Transformer", "FlatGradBucket", "HubertWithKmeans",
           "EncodecWrapper", "FairseqVQWav2Vec"]
