"""hnswlib-rs_b200 — H100-native HNSW search/insert engine behind the hnsw_rs API surface.

The product is hnswlib-rs_b200/lib/libhnsw_b200.so (C ABI in include/hnsw_b200.h, CUDA sm_90a).
This package is the thin host-side mirror of the reference's interface over that ABI.
The directory name contains '-': import it with importlib.import_module("hnswlib-rs_b200").
"""
from .hnsw import ATTR_NONE, LABEL_NONE, RANGE_ALL, Hnsw, HnswError, Neighbour, ResidentFilter, last_error, last_kernel, last_kernel_shape, lib_path, load_library, attr_of_float  # noqa: F401
from . import datagen  # noqa: F401
