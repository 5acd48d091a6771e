"""minio_b200 — H100-native (sm_90a) erasure-code + bitrot hot path of MinIO (RS GF(2^8) + HighwayHash-256).

The product is the C-ABI shared library ``libminio_ec.so`` (include/minio_ec.h) built from
``minio_b200/csrc``; this package is only the thin ctypes binding tests and bench.py use.
There is no CPU implementation here: without the built CUDA library, importing fails loudly.
"""
from . import capi
from .capi import (BLAKE2B512, HIGHWAYHASH256, HIGHWAYHASH256S, SHA256, Batcher, Codec, MecError, device_count, lib,
                   lib_path, heal_batch, pinned_array, selftest)

__all__ = ["Codec", "Batcher", "capi", "MecError", "lib", "lib_path", "device_count", "selftest", "SHA256", "HIGHWAYHASH256",
           "HIGHWAYHASH256S", "BLAKE2B512", "heal_batch", "pinned_array"]
