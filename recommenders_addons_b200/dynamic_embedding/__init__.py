"""Mirror of the reference's `tfra.dynamic_embedding` export list for the hot path
(/root/reference/tensorflow_recommenders_addons/dynamic_embedding/__init__.py:17-53)."""
from .table import (CuckooHashTable, CuckooHashTableConfig, CuckooHashTableCreator, DynamicEmbeddingSaver,
                    FileSystemSaver, FileSystemSaverConfig, HkvEvictStrategy, HkvHashTable, HkvHashTableConfig,
                    HkvHashTableCreator, KVCreator)
from .variable import (GraphKeys, ModelMode, TrainableWrapper, Variable, default_partition_fn, embedding_lookup,
                       embedding_lookup_unique, enable_inference_mode, enable_train_mode, get_model_mode, get_variable,
                       load_de_variable_from_file_system, make_partition, segment_reduce, trainable_wrapper_filter, unique)
from .keyed_init import KeyedRandomNormal, KeyedRandomUniform, KeyedTruncatedNormal
from .ops import (SparseIds, SparseLookupTrainable, embedding_lookup_sparse, safe_embedding_lookup_sparse,
                  trainable_embedding_lookup_sparse, trainable_safe_embedding_lookup_sparse)
from .optimizer import (ComposedOptimizer, DynamicEmbeddingOptimizer, FusedAdadelta, FusedAdagrad, FusedAdagradDA,
                        FusedAdam, FusedAdamax, FusedAdamW, FusedFtrl, FusedLion, FusedNadam, FusedProximalAdagrad,
                        FusedProximalGradientDescent, FusedRMSprop, FusedSGD, SlotPlane)
from .restrict_policies import FrequencyRestrictPolicy, RestrictPolicy, TimestampRestrictPolicy
from .sharded import PeerShardedVariable, ShardedVariable
from . import layers
from . import shadow_ops
from . import math
from . import data_flow
from . import keras

__all__ = [
    "CuckooHashTable", "CuckooHashTableConfig", "CuckooHashTableCreator", "HkvEvictStrategy", "HkvHashTable", "HkvHashTableConfig",
    "HkvHashTableCreator", "KVCreator", "Variable", "default_partition_fn", "embedding_lookup",
    "embedding_lookup_unique", "get_variable", "unique", "segment_reduce", "SparseIds", "embedding_lookup_sparse",
    "safe_embedding_lookup_sparse", "DynamicEmbeddingOptimizer", "FusedAdagrad", "FusedAdam", "FusedSGD", "FusedFtrl", "FusedRMSprop", "FusedAdadelta", "FusedAdamax", "FusedNadam", "FusedProximalAdagrad", "FusedProximalGradientDescent", "FusedAdagradDA", "FusedAdamW", "FusedLion", "ShardedVariable", "PeerShardedVariable", "layers",
    "RestrictPolicy", "TimestampRestrictPolicy", "FrequencyRestrictPolicy", "TrainableWrapper", "ModelMode",
    "enable_inference_mode", "enable_train_mode", "get_model_mode", "trainable_wrapper_filter", "shadow_ops",
    "ComposedOptimizer", "SlotPlane", "math", "data_flow", "keras", "GraphKeys", "FileSystemSaver", "FileSystemSaverConfig", "DynamicEmbeddingSaver",
    "KeyedRandomNormal", "KeyedRandomUniform", "KeyedTruncatedNormal", "SparseLookupTrainable",
    "trainable_embedding_lookup_sparse", "trainable_safe_embedding_lookup_sparse",
]
