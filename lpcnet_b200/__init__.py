"""lpcnet_b200 — H100-native LPCNet synthesis engine (host-side Python mirror of the C ABI).

The product is `liblpcnet_b200.so` (C host + sm_90a CUDA kernels, include/lpcnet.h + include/lpcnet_b200.h).
This package only loads it through ctypes and mirrors the reference's operator interface
(`lpcnet_create/lpcnet_load_model/lpcnet_synthesize/lpcnet_decode`, reference include/lpcnet.h) plus the batched
extension, so that tests and the benchmark read like calls into the reference library.  There is no Python
compute path and no CPU fallback: without the built library or without a CUDA device every call raises.
"""
from .api import (Batch, Group, group_plan, group_plan_float, mixed_plan, MixedGroup, Multi, MultiGroup, EncBatch, LPCNet, LPCNetDecoder, lib, LPCNetB200Error, device_count, measure_smem_peak,  # noqa: F401
                  parse_blob, write_blob, blob_config, shard_range)
