"""dib_b200 -- H100-native Distributed Information Bottleneck training engine.

Drop-in for the hot path of distributed-information-bottleneck.github.io: ``models.DistributedIBNet`` /
``model.compile`` / ``model.fit`` / ``InfoBottleneckAnnealingCallback`` / ``SaveCompressionMatricesCallback``,
backed by hand-written sm_90a CUDA kernels behind the C ABI of include/dib_b200.h.
"""
from . import ctw, keras_compat, metrics, models, parallel, utils                     # noqa: F401
from .keras_compat import Adam, SGD, RMSprop, Callback, History, losses, optimizers           # noqa: F401
from .models import (DistributedIBNet, InfoBottleneckAnnealingCallback, PositionalEncoding,   # noqa: F401
                     SaveCompressionMatricesCallback, StashEmbeddingsCallback, InfoPerFeatureCallback,
                     ParticleInformationCallback, SimpleEncoder, SharedParticleEncoder, SetTransformerIBNet, pad_sets)
from ._lib import DibError, library_path                                         # noqa: F401

__all__ = ["DistributedIBNet", "PositionalEncoding", "InfoBottleneckAnnealingCallback",
           "SaveCompressionMatricesCallback", "StashEmbeddingsCallback", "InfoPerFeatureCallback",
           "ParticleInformationCallback", "SimpleEncoder",
           "SharedParticleEncoder", "SetTransformerIBNet", "pad_sets", "Adam", "SGD", "RMSprop", "optimizers", "losses",
           "Callback", "History", "models", "metrics", "utils", "parallel", "keras_compat", "DibError", "library_path"]
