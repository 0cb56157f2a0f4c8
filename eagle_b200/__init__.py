"""eagle_b200: an H100-native (sm_90a) engine for EAGLE speculative decoding.

`EaModel` keeps the reference's API (SafeAILab/EAGLE eagle/model/ea_model.py) and checkpoint
format; the draft -> verify -> accept cycle runs in libeagle_b200.so (include/eagle_b200.h).
"""
from .ea_model import EaModel, static_tree_buffers  # noqa: F401

__all__ = ["EaModel", "static_tree_buffers"]
