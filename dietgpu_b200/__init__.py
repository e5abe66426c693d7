"""dietgpu_b200 -- H100-native batched rANS + float codec behind DietGPU's API.

The package is a thin host layer over libdietgpu_b200.so (hand-written sm_90a
CUDA, C ABI in include/dietgpu_b200.h).  There is no CPU fallback: the first
call that needs the library raises ImportError if it has not been built.
"""
from . import capi  # noqa: F401
from .host import HostCodec  # noqa: F401
from .collectives import (  # noqa: F401
    PeerWorkspace,
    all_gather_compressed,
    all_reduce_compressed,
    all_to_all_compressed,
    exchange_archives,
    reduce_scatter_compressed,
)
from .ops import (  # noqa: F401
    compress_data,
    compress_data_simple,
    compress_data_split_size,
    decompress_data,
    decompress_data_reduce,
    decompress_data_simple,
    decompress_data_split_size,
    max_any_compressed_output_size,
    max_any_compressed_size,
    max_float_compressed_output_size,
    max_float_compressed_size,
    sq_norm,
)

__all__ = [
    "capi", "HostCodec", "PeerWorkspace", "all_gather_compressed", "all_to_all_compressed", "exchange_archives",
    "reduce_scatter_compressed", "all_reduce_compressed", "decompress_data_reduce", "compress_data", "compress_data_simple", "compress_data_split_size", "decompress_data",
    "decompress_data_simple", "decompress_data_split_size", "max_any_compressed_output_size",
    "max_any_compressed_size", "max_float_compressed_output_size", "max_float_compressed_size", "sq_norm",
]
