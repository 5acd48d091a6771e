"""ctypes binding of include/minio_ec.h.  Host buffers are numpy uint8 arrays; device buffers are
raw pointers (e.g. ``torch.Tensor.data_ptr()``)."""
import ctypes as C
import os

import numpy as np

SHA256, HIGHWAYHASH256, HIGHWAYHASH256S, BLAKE2B512 = 1, 2, 3, 4
ERRORS = {-1: "ErrInvShardNum", -2: "ErrMaxShardNum", -3: "ErrTooFewShards", -4: "ErrShardNoData", -5: "ErrShardSize",
          -6: "ErrShortData", -7: "errFileCorrupt", -8: "errLessData", -9: "errUnexpected", -10: "errErasureReadQuorum",
          -11: "errErasureWriteQuorum", -12: "errInvalidArgument", -13: "sio.NotAuthentic (errObjectTampered)", -14: "errSignatureMismatch",
          -15: "errMalformedEncoding", -16: "errChunkTooBig", -17: "io.ErrUnexpectedEOF (IncompleteBody)", -18: "ioutil.ErrOverread", -100: "CUDA error", -101: "no CUDA device",
          -102: "unsupported on the GPU path"}
MIX_PATTERNS = 1  # MEC_BATCHER_MIX_PATTERNS
CRC32, CRC32C, CRC64NVME = 1, 2, 4  # MEC_CRC*
SUM_MD5, SUM_SHA1, SUM_SHA256 = 8, 16, 32  # MEC_SUM_*
DARE_SEAL, DARE_OPEN = 1, 2  # MEC_DARE_*
NOT_AUTHENTIC = -13  # MEC_ERR_NOT_AUTHENTIC
# MEC_ERR_* of Signature V4 streaming bodies (mec_encode_chunked)
SIGNATURE_MISMATCH, MALFORMED_ENCODING, CHUNK_TOO_BIG, INCOMPLETE_BODY, OVERREAD = -14, -15, -16, -17, -18
SIGV4_PAYLOAD, SIGV4_TRAILER = 0, 1  # MEC_SIGV4_*
SUM_BYTES = 96  # MEC_SUM_BYTES: one record of mec_sums_device / mec_batcher_encode_sums
SUM_SLOTS = {"md5": (SUM_MD5, 0, 16), "sha1": (SUM_SHA1, 32, 20), "sha256": (SUM_SHA256, 64, 32)}  # name -> (bit, offset, length)

_LIB = None


class MecError(RuntimeError):
    def __init__(self, code, what=""):
        self.code = code
        detail = lib().mec_last_error().decode() if code <= -100 else ""
        super().__init__(f"{what}: {ERRORS.get(code, code)} ({code}) {detail}")


def lib_path():
    # MEC_LIB selects an experimental build variant (tools/build_variants.sh); default is the product library
    return os.environ.get("MEC_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "libminio_ec.so")


def lib():
    """Load libminio_ec.so.  Fails loudly when the CUDA extension has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        raise RuntimeError(f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
    L = C.CDLL(path)
    vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int
    L.mec_codec_new.argtypes = [i32, i32, i64, i32, i32, C.POINTER(vp)]
    L.mec_codec_free.argtypes = [vp]
    L.mec_codec_free.restype = None
    L.mec_last_error.restype = C.c_char_p
    L.mec_version.restype = C.c_char_p
    for f, args in (("mec_shard_size", [vp]), ("mec_shard_file_size", [vp, i64]),
                    ("mec_shard_file_offset", [vp, i64, i64, i64]), ("mec_bitrot_shard_file_size", [i64, i64, i32]),
                    ("mec_ceil_frac", [i64, i64]), ("mec_launch_count", [vp])):
        getattr(L, f).restype = i64
        getattr(L, f).argtypes = args
    L.mec_alloc_pinned.restype = vp
    L.mec_alloc_pinned.argtypes = [C.c_size_t]
    L.mec_free_pinned.argtypes = [vp]
    L.mec_free_pinned.restype = None
    L.mec_alloc_pinned_on.restype = vp
    L.mec_alloc_pinned_on.argtypes = [i32, C.c_size_t]
    L.mec_device_numa_node.argtypes = [i32]
    L.mec_bind_thread_to_device.argtypes = [i32]
    L.mec_is_pinned.argtypes = [vp]
    L.mec_encode_sg.restype = i64
    L.mec_encode_sg.argtypes = [vp, vp, i64, vp, vp, i32]
    L.mec_heal_prefer.argtypes = [vp, vp, vp, i64, vp, vp]
    L.mec_batcher_new.argtypes = [i32, i32, i64, i32, i64, i32, C.POINTER(vp)]
    L.mec_batcher_new_ex.argtypes = [i32, i32, i64, i32, i64, i32, i32, C.POINTER(vp)]
    L.mec_batcher_free.argtypes = [vp]
    L.mec_batcher_free.restype = None
    L.mec_batcher_encode.restype = i64
    L.mec_batcher_encode.argtypes = [vp, vp, i64, vp, i32]
    L.mec_batcher_encode_sg.restype = i64
    L.mec_batcher_encode_sg.argtypes = [vp, vp, i64, vp, vp, i32]
    L.mec_batcher_encode_crc.restype = i64
    L.mec_batcher_encode_crc.argtypes = [vp, vp, i64, vp, vp, i32, i32, vp]
    L.mec_batcher_encode_sums.restype = i64
    L.mec_batcher_encode_sums.argtypes = [vp, vp, i64, vp, vp, i32, i32, vp, vp]
    L.mec_sums_device.argtypes = [vp, i32, vp, vp, vp, i64, vp, vp]
    L.mec_batcher_decode.restype = i64
    L.mec_batcher_decode.argtypes = [vp, vp, i64, i64, i64, vp, C.POINTER(i32)]
    L.mec_batcher_decode_prefer.restype = i64
    L.mec_batcher_decode_prefer.argtypes = [vp, vp, vp, i64, i64, i64, vp, C.POINTER(i32)]
    L.mec_batcher_heal.argtypes = [vp, vp, vp, i64, vp, vp]
    L.mec_batcher_new_transcode.argtypes = [i32, i32, i32, i32, i64, i32, i64, i32, i32, C.POINTER(vp)]
    L.mec_batcher_new_transcode_ex.argtypes = [i32, i32, i64, i32, i32, i64, i32, i64, i32, i32, C.POINTER(vp)]
    L.mec_batcher_transcode.restype = i64
    L.mec_batcher_transcode.argtypes = [vp, vp, vp, i64, vp, i32, C.POINTER(i32)]
    L.mec_batcher_transcode_whole.restype = i64
    L.mec_batcher_transcode_whole.argtypes = [vp, i32, vp, vp, vp, i64, vp, i32, C.POINTER(i32)]
    L.mec_batcher_decode_mixed.restype = i64
    L.mec_batcher_decode_mixed.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, vp, C.POINTER(i32)]
    L.mec_batcher_heal_mixed.argtypes = [vp, vp, vp, vp, vp, i64, vp, vp]
    L.mec_batcher_stat.restype = i64
    L.mec_batcher_stat.argtypes = [vp, C.c_char_p]
    L.mec_batcher_set_option.argtypes = [vp, C.c_char_p, i64]
    L.mec_checksums.argtypes = [vp, vp, i64, i32, vp]
    L.mec_checksums_device.argtypes = [vp, vp, i64, i32, vp, vp]
    L.mec_checksum_combine.restype = C.c_uint64
    L.mec_checksum_combine.argtypes = [i32, C.c_uint64, C.c_uint64, i64]
    L.mec_last_checksums.restype = i64
    L.mec_last_checksums.argtypes = [vp, vp]
    L.mec_decode_whole.restype = i64
    L.mec_decode_whole.argtypes = [vp, vp, vp, i64, i64, i64, vp, C.POINTER(i32)]
    L.mec_heal_whole.argtypes = [vp, vp, vp, i64, vp, vp, vp]
    L.mec_decode_mixed.restype = i64
    L.mec_decode_mixed.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, vp, C.POINTER(i32)]
    L.mec_heal_mixed.argtypes = [vp, vp, vp, vp, vp, i64, vp, vp]
    L.mec_encode_blocks.argtypes = [vp, vp, i64, vp, vp]
    L.mec_encode_blocks_device.argtypes = [vp, vp, i64, vp, i64, vp, vp]
    L.mec_reconstruct_frames.argtypes = [vp, vp, i64, i64, vp, i32, vp, vp]
    L.mec_reconstruct_device.argtypes = [vp, vp, i64, i64, vp, i32, vp, i64, vp, vp, vp]
    L.mec_encode.restype = i64
    L.mec_encode.argtypes = [vp, vp, i64, vp, i32]
    L.mec_decode.restype = i64
    L.mec_decode.argtypes = [vp, vp, i64, i64, i64, vp, C.POINTER(i32)]
    L.mec_heal.argtypes = [vp, vp, i64, vp]
    L.mec_heal_batch.argtypes = [vp, i32, i64, vp, vp, vp, vp]
    L.mec_decode_prefer.restype = i64
    L.mec_decode_prefer.argtypes = [vp, vp, vp, i64, i64, i64, vp, C.POINTER(i32)]
    L.mec_transcode.restype = i64
    L.mec_transcode.argtypes = [vp, vp, vp, i64, vp, vp, i32, C.POINTER(i32)]
    L.mec_transcode_whole.restype = i64
    L.mec_transcode_whole.argtypes = [vp, vp, vp, vp, i64, vp, vp, i32, C.POINTER(i32)]
    L.mec_jit_compile_check.restype = i64
    L.mec_jit_compile_check.argtypes = [i32, i32, vp, i32, i32, i32, i32]
    L.mec_jit_prewarm.argtypes = [vp]
    L.mec_shutdown.restype = None
    L.mec_shutdown.argtypes = []
    import atexit
    atexit.register(L.mec_shutdown)  # no NVRTC compile may be in flight when the C runtime starts its exit handlers
    L.mec_get_stat.restype = i64
    L.mec_get_stat.argtypes = [vp, C.c_char_p]
    L.mec_bitrot_verify.argtypes = [vp, vp, i64, i64]
    L.mec_bitrot_verify_batch.argtypes = [vp, i64, vp, vp, vp, vp]
    L.mec_bitrot_verify_parts.argtypes = [vp, i64, vp, vp, vp, vp, vp, C.POINTER(i32)]
    L.mec_batcher_verify.argtypes = [vp, i64, vp, vp, vp, vp, vp, C.POINTER(i32)]
    L.mec_encode_whole.restype = i64
    L.mec_encode_whole.argtypes = [vp, vp, i64, vp, vp, i32]
    L.mec_whole_hash.argtypes = [vp, i32, vp, i64, i64, vp]
    L.mec_bitrot_verify_whole.argtypes = [vp, i32, vp, i64, vp]
    L.mec_digest_size.argtypes = [i32]
    L.mec_whole_hash_device.argtypes = [vp, i32, vp, i64, i64, i64, vp, vp]
    L.mec_rs_encode_shards.argtypes = [vp, vp, i64]
    L.mec_rs_reconstruct_shards.argtypes = [vp, vp, vp, i64, i32]
    L.mec_hh256_batch.argtypes = [vp, vp, i64, i64, vp]
    L.mec_selftest.argtypes = [i32]
    L.mec_set_option.argtypes = [vp, C.c_char_p, i64]
    for f in ("mec_dare_encrypted_size", "mec_dare_decrypted_size"):
        getattr(L, f).restype = i64
        getattr(L, f).argtypes = [i64]
    L.mec_dare_device.argtypes = [vp, i32, i64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.mec_encode_sse.restype = i64
    L.mec_encode_sse.argtypes = [vp, vp, i64, vp, vp, vp, i32]
    L.mec_decode_sse.restype = i64
    L.mec_decode_sse.argtypes = [vp, vp, vp, i64, i64, i64, vp, vp, C.POINTER(i32)]
    L.mec_batcher_encode_sse.restype = i64
    L.mec_batcher_encode_sse.argtypes = [vp, vp, i64, vp, vp, vp, i32]
    L.mec_batcher_decode_sse.restype = i64
    L.mec_batcher_decode_sse.argtypes = [vp, vp, vp, i64, i64, i64, vp, vp, C.POINTER(i32)]
    L.mec_chunk_signatures_device.argtypes = [vp, vp, C.c_char_p, C.c_char_p, vp, vp, vp, vp, vp, vp, i64, vp, vp]
    L.mec_encode_chunked.restype = i64
    L.mec_encode_chunked.argtypes = [vp, vp, i64, i64, vp, vp, C.c_char_p, C.c_char_p, i32, vp, i32, vp, i64, C.POINTER(i64)]
    L.mec_encode_chunked_sse.restype = i64
    L.mec_encode_chunked_sse.argtypes = [vp, vp, i64, i64, vp, vp, C.c_char_p, C.c_char_p, i32, vp, vp, vp, i32, vp, i64,
                                         C.POINTER(i64)]
    _LIB = L
    return L


def device_count():
    return lib().mec_device_count()


def selftest(device=0):
    rc = lib().mec_selftest(device)
    if rc:
        raise MecError(rc, "mec_selftest")


def _u8(a):
    if isinstance(a, (bytes, bytearray, memoryview)):
        a = np.frombuffer(a, dtype=np.uint8)
    a = np.ascontiguousarray(a, dtype=np.uint8)
    return a


def _ptrs(arrs):
    return (C.c_void_p * len(arrs))(*[(a.ctypes.data if (a is not None and a.size) else None) for a in arrs])


def _verify_parts(fn, h, what, files, algos, part_lens, sums):
    """the shared body of Codec.bitrot_verify_parts and Batcher.verify"""
    files = [None if f is None else _u8(f) for f in files]
    n = len(files)
    al = (C.c_int32 * max(n, 1))(*[int(a) for a in algos])
    fl = (C.c_int64 * max(n, 1))(*[0 if f is None else f.size for f in files])
    pl = (C.c_int64 * max(n, 1))(*[int(x) for x in part_lens])
    sm = None
    if sums is not None:
        sm = np.zeros((max(n, 1), 64), dtype=np.uint8)
        for i, d in enumerate(sums):
            if d is not None:
                sm[i, :len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
    res = (C.c_int32 * max(n, 1))()
    rc = fn(h, n, al, _ptrs(files) if n else (C.c_void_p * 1)(), fl, pl, None if sm is None else sm.ctypes.data, res)
    if rc:
        raise MecError(rc, what)
    return list(res)[:n]


class Codec:
    """NewErasure (cmd/erasure-coding.go:42) bound to one CUDA device."""

    def __init__(self, k, m, block_size=1 << 20, algo=HIGHWAYHASH256S, device=0):
        h = C.c_void_p()
        rc = lib().mec_codec_new(k, m, block_size, algo, device, C.byref(h))
        if rc:
            raise MecError(rc, "mec_codec_new")
        self.h, self.k, self.m, self.n, self.block_size, self.algo = h, k, m, k + m, block_size, algo

    def close(self):
        if getattr(self, "h", None):
            lib().mec_codec_free(self.h)
            self.h = None

    __del__ = close

    # -- helpers
    def set_option(self, name, value):
        rc = lib().mec_set_option(self.h, name.encode(), int(value))
        if rc:
            raise MecError(rc, "mec_set_option")

    @property
    def launches(self):
        return lib().mec_launch_count(self.h)

    def shard_size(self):
        return lib().mec_shard_size(self.h)

    def shard_file_size(self, total):
        return lib().mec_shard_file_size(self.h, total)

    def shard_file_offset(self, start, length, total):
        return lib().mec_shard_file_offset(self.h, start, length, total)

    def bitrot_file_size(self, total):
        return lib().mec_bitrot_shard_file_size(self.shard_file_size(total), self.shard_size(), self.algo)

    # -- block level
    def encode_blocks(self, src):
        """-> (parity [nblocks, m, S], digests [nblocks, n, 32]); the last block may use < S bytes per row."""
        src = _u8(src)
        nb = -(-src.size // self.block_size)
        S = self.shard_size()
        parity = np.zeros((nb, max(self.m, 1), S), dtype=np.uint8)
        dig = np.zeros((nb, self.n, 32), dtype=np.uint8)
        rc = lib().mec_encode_blocks(self.h, src.ctypes.data if src.size else None, src.size, parity.ctypes.data, dig.ctypes.data)
        if rc:
            raise MecError(rc, "mec_encode_blocks")
        return parity[:, :self.m], dig

    def encode_blocks_device(self, d_src, length, d_parity, parity_pitch, d_digests, stream=0):
        rc = lib().mec_encode_blocks_device(self.h, d_src, length, d_parity, parity_pitch, d_digests, stream)
        if rc:
            raise MecError(rc, "mec_encode_blocks_device")

    def reconstruct_device(self, d_frames, frame_pitch, nblocks, want, data_only, d_out, out_pitch, d_digests, d_corrupt, stream=0):
        """d_frames: list of k+m device pointers (0/None = unavailable).  data_only: bool, or the MEC_RECONSTRUCT_* flag bits
        (1 = data only, 2 = no digests for the rebuilt shards)."""
        arr = (C.c_void_p * self.n)(*[(p or None) for p in d_frames])
        want = np.asarray(want, dtype=np.uint8)
        rc = lib().mec_reconstruct_device(self.h, arr, frame_pitch, nblocks, want.ctypes.data, int(data_only),
                                          d_out, out_pitch, d_digests, d_corrupt, stream)
        if rc:
            raise MecError(rc, "mec_reconstruct_device")

    # -- whole part
    def encode(self, src, online=None, write_quorum=0):
        src = _u8(src)
        fsz = self.bitrot_file_size(src.size)
        online = [True] * self.n if online is None else online
        files = [np.zeros(fsz, dtype=np.uint8) if online[i] else None for i in range(self.n)]
        rc = lib().mec_encode(self.h, src.ctypes.data if src.size else None, src.size, _ptrs(files), write_quorum)
        if rc < 0:
            raise MecError(rc, "mec_encode")
        return files

    def encode_sg(self, src, online=None, write_quorum=0):
        """mec_encode_sg: -> (files, data_digests).  files[i] is None for data drives (their frames are the caller's own
        source slices behind data_digests[b, i]) and the complete part.N image for online parity drives."""
        src = _u8(src)
        fsz = self.bitrot_file_size(src.size)
        nb = -(-src.size // self.block_size)
        online = [True] * self.n if online is None else online
        marker = np.zeros(1, dtype=np.uint8)  # data drives: only NULL / non-NULL is looked at
        files = [(np.zeros(fsz, dtype=np.uint8) if i >= self.k else marker) if online[i] else None for i in range(self.n)]
        dd = np.zeros((max(nb, 1), self.k, 32), dtype=np.uint8)
        rc = lib().mec_encode_sg(self.h, src.ctypes.data if src.size else None, src.size, _ptrs(files), dd.ctypes.data, write_quorum)
        if rc < 0:
            raise MecError(rc, "mec_encode_sg")
        return [f if i >= self.k else None for i, f in enumerate(files)], dd[:nb]

    def checksums(self, data, which=7):
        """-> (CRC32, CRC32C, CRC64NVME) of a host byte string (mec_checksums); 0 where not asked for."""
        d = _u8(data)
        out = (C.c_uint64 * 3)()
        rc = lib().mec_checksums(self.h, d.ctypes.data if d.size else None, d.size, which, out)
        if rc:
            raise MecError(rc, "mec_checksums")
        return tuple(int(v) for v in out)

    def checksums_device(self, d_src, length, which=7, stream=0):
        out = (C.c_uint64 * 3)()
        rc = lib().mec_checksums_device(self.h, d_src, length, which, out, stream)
        if rc:
            raise MecError(rc, "mec_checksums_device")
        return tuple(int(v) for v in out)

    def sums_device(self, d_base, offsets, lens, which, d_sums, stream=0):
        """mec_sums_device: MD5 / SHA-1 / SHA-256 (a mask of SUM_*) of the messages d_base[offsets[i], offsets[i] + lens[i]) in device
        memory; record i (SUM_BYTES bytes, see SUM_SLOTS) at d_sums + i * SUM_BYTES.  Asynchronous on `stream`."""
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        ln = np.ascontiguousarray(lens, dtype=np.int64)
        if off.size != ln.size:
            raise ValueError("offsets and lens differ in length")
        rc = lib().mec_sums_device(self.h, which, d_base, off.ctypes.data, ln.ctypes.data, off.size, d_sums, stream)
        if rc:
            raise MecError(rc, "mec_sums_device")

    def last_checksums(self):
        out = (C.c_uint64 * 3)()
        n = lib().mec_last_checksums(self.h, out)
        return tuple(int(v) for v in out), n

    def stat(self, name):
        return lib().mec_get_stat(self.h, name.encode())

    # -- server-side encryption (DARE 2.0, AES-256-GCM)
    def encode_sse(self, src, key, nonce, online=None, write_quorum=0):
        """mec_encode_sse -> part files"""
        src, key, nonce = _u8(src), _u8(key), _u8(nonce)
        if key.size != 32 or nonce.size != 12:
            raise ValueError("key is 32 bytes, nonce 12")
        enc = dare_encrypted_size(src.size)
        fsz = self.bitrot_file_size(enc)
        online = [True] * self.n if online is None else online
        files = [np.zeros(fsz, dtype=np.uint8) if online[i] else None for i in range(self.n)]
        rc = lib().mec_encode_sse(self.h, src.ctypes.data if src.size else None, src.size, key.ctypes.data, nonce.ctypes.data,
                                  _ptrs(files), write_quorum)
        if rc < 0:
            raise MecError(rc, "mec_encode_sse")
        return files

    def decode_sse(self, files, offset, length, enc_total, key, prefer=None):
        """mec_decode_sse -> (plaintext [offset, offset + length), heal_hint)"""
        files = [None if f is None else _u8(f) for f in files]
        key = _u8(key)
        if key.size != 32:
            raise ValueError("key is 32 bytes")
        dst = np.zeros(max(length, 1), dtype=np.uint8)
        hint = C.c_int(0)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        rc = lib().mec_decode_sse(self.h, _ptrs(files), None if pf is None else pf.ctypes.data, offset, length, enc_total,
                                  key.ctypes.data, dst.ctypes.data, C.byref(hint))
        if rc < 0:
            raise MecError(rc, "mec_decode_sse")
        return dst[:length], hint.value

    def dare_device(self, op, keys, d_in, in_off, lens, d_out, out_off, seq0=None, nonces=None, enc_totals=None, stream=0,
                    check=True):
        """mec_dare_device over len(lens) streams -> (rc, per-stream status); check=True raises MecError on rc != 0"""
        ns = len(lens)
        keys = np.ascontiguousarray(keys, dtype=np.uint8).reshape(ns, 32)
        seq = np.zeros(ns, dtype=np.uint32) if seq0 is None else np.ascontiguousarray(seq0, dtype=np.uint32)
        arr = {name: np.ascontiguousarray(v, dtype=np.int64) for name, v in (("in", in_off), ("lens", lens), ("out", out_off))}
        nn = None if nonces is None else np.ascontiguousarray(nonces, dtype=np.uint8).reshape(ns, 12)
        et = None if enc_totals is None else np.ascontiguousarray(enc_totals, dtype=np.int64)
        status = np.zeros(max(ns, 1), dtype=np.uint8)
        rc = lib().mec_dare_device(self.h, op, ns, keys.ctypes.data, None if nn is None else nn.ctypes.data, seq.ctypes.data,
                                   None if et is None else et.ctypes.data, d_in, arr["in"].ctypes.data, arr["lens"].ctypes.data,
                                   d_out, arr["out"].ctypes.data, status.ctypes.data, stream)
        if check and rc:
            raise MecError(rc, "mec_dare_device")
        return rc, status[:ns]

    # -- Signature V4 streaming payloads (aws-chunked bodies)
    def chunk_signatures_device(self, key, date, scope, d_base, offsets, lens, prev, claimed, kinds, stream=0):
        """mec_chunk_signatures_device over len(lens) rows in ONE launch -> verdicts (1 = the claimed signature matches).
        prev / claimed: 64 bytes per row (bytes objects or an (n, 64) uint8 array); kinds: SIGV4_PAYLOAD / SIGV4_TRAILER."""
        n = len(lens)
        key = _u8(key)
        if key.size != 32:
            raise ValueError("the signing key is 32 bytes")
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        ln = np.ascontiguousarray(lens, dtype=np.int64)
        pv = np.frombuffer(b"".join(prev), dtype=np.uint8) if isinstance(prev, (list, tuple)) else _u8(prev)
        cl = np.frombuffer(b"".join(claimed), dtype=np.uint8) if isinstance(claimed, (list, tuple)) else _u8(claimed)
        kd = np.ascontiguousarray(kinds, dtype=np.int32)
        if not (off.size == ln.size == kd.size == n and pv.size == cl.size == 64 * n):
            raise ValueError("one offset, length, kind and 64-byte previous and claimed signature per row")
        out = np.zeros(max(n, 1), dtype=np.uint8)
        rc = lib().mec_chunk_signatures_device(self.h, key.ctypes.data, date.encode(), scope.encode(), d_base, off.ctypes.data,
                                               ln.ctypes.data, pv.ctypes.data, cl.ctypes.data, kd.ctypes.data, n, out.ctypes.data,
                                               stream)
        if rc:
            raise MecError(rc, "mec_chunk_signatures_device")
        return out[:n]

    def encode_chunked(self, body, decoded_len, key, seed, date, scope, trailer=False, online=None, write_quorum=0,
                       trailer_cap=4096):
        """mec_encode_chunked: an aws-chunked body -> part files of its decoded_len decoded bytes; with trailer=True
        (part files, trailer value as signed)"""
        body, key = _u8(body), _u8(key)
        seed = seed if isinstance(seed, bytes) else bytes(_u8(seed))
        if key.size != 32 or len(seed) != 64:
            raise ValueError("the signing key is 32 bytes, the seed signature 64")
        fsz = self.bitrot_file_size(decoded_len) if decoded_len > 0 else 0
        online = [True] * self.n if online is None else online
        files = [np.zeros(fsz, dtype=np.uint8) if online[i] else None for i in range(self.n)]
        sd = np.frombuffer(seed, dtype=np.uint8)
        tout = np.zeros(max(trailer_cap, 1), dtype=np.uint8)
        tlen = C.c_int64(0)
        rc = lib().mec_encode_chunked(self.h, body.ctypes.data if body.size else None, body.size, decoded_len, key.ctypes.data,
                                      sd.ctypes.data, date.encode(), scope.encode(), int(trailer), _ptrs(files), write_quorum,
                                      tout.ctypes.data, trailer_cap, C.byref(tlen))
        if rc < 0:
            raise MecError(rc, "mec_encode_chunked")
        if trailer:
            return files, bytes(tout[:min(tlen.value, trailer_cap)])
        return files

    def encode_chunked_sse(self, body, decoded_len, key, seed, date, scope, sse_key, nonce, trailer=False, online=None,
                           write_quorum=0, trailer_cap=4096):
        """mec_encode_chunked_sse: an aws-chunked body of an encrypted bucket -> the part files encode_sse writes for its decoded_len
        decoded bytes; with trailer=True (part files, trailer value as signed)"""
        body, key, sse_key, nonce = _u8(body), _u8(key), _u8(sse_key), _u8(nonce)
        seed = seed if isinstance(seed, bytes) else bytes(_u8(seed))
        if key.size != 32 or len(seed) != 64:
            raise ValueError("the signing key is 32 bytes, the seed signature 64")
        if sse_key.size != 32 or nonce.size != 12:
            raise ValueError("the SSE key is 32 bytes, the nonce 12")
        fsz = self.bitrot_file_size(dare_encrypted_size(decoded_len)) if decoded_len > 0 else 0
        online = [True] * self.n if online is None else online
        files = [np.zeros(fsz, dtype=np.uint8) if online[i] else None for i in range(self.n)]
        sd = np.frombuffer(seed, dtype=np.uint8)
        tout = np.zeros(max(trailer_cap, 1), dtype=np.uint8)
        tlen = C.c_int64(0)
        rc = lib().mec_encode_chunked_sse(self.h, body.ctypes.data if body.size else None, body.size, decoded_len, key.ctypes.data,
                                          sd.ctypes.data, date.encode(), scope.encode(), int(trailer), sse_key.ctypes.data,
                                          nonce.ctypes.data, _ptrs(files), write_quorum, tout.ctypes.data, trailer_cap, C.byref(tlen))
        if rc < 0:
            raise MecError(rc, "mec_encode_chunked_sse")
        if trailer:
            return files, bytes(tout[:min(tlen.value, trailer_cap)])
        return files

    def decode(self, files, offset, length, total, prefer=None):
        files = [None if f is None else _u8(f) for f in files]
        dst = np.zeros(max(length, 1), dtype=np.uint8)
        hint = C.c_int(0)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        rc = lib().mec_decode_prefer(self.h, _ptrs(files), None if pf is None else pf.ctypes.data, offset, length, total,
                                     dst.ctypes.data, C.byref(hint))
        if rc < 0:
            raise MecError(rc, "mec_decode")
        return dst[:length], hint.value

    def transcode(self, files, total, dst, prefer=None, online=None, write_quorum=0):
        """mec_transcode: move a whole part of `total` bytes from this codec's part files (None = offline) to the geometry of the
        Codec `dst` without the object bytes leaving the device.  online = dst's writers (None = all).  -> (out_files, heal_hint):
        dst's complete part files (None where offline) and -7 when a source frame failed its digest on the way."""
        files = [None if f is None else _u8(f) for f in files]
        fsz = dst.bitrot_file_size(total)
        online = [True] * dst.n if online is None else online
        outs = [np.zeros(fsz, dtype=np.uint8) if online[i] else None for i in range(dst.n)]
        hint = C.c_int(0)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        # an empty part has empty out files, yet an online writer must still count against the quorum
        marker = np.zeros(1, dtype=np.uint8)
        optrs = _ptrs([(o if o.size else marker) if o is not None else None for o in outs])
        rc = lib().mec_transcode(self.h, _ptrs(files), None if pf is None else pf.ctypes.data, total, dst.h, optrs, write_quorum,
                                 C.byref(hint))
        if rc < 0:
            raise MecError(rc, "mec_transcode")
        return outs, hint.value

    def heal(self, files, stale, total, prefer=None, report=False):
        """Erasure.Heal.  Like the reference, bitrot met in a source reader does not stop the rebuild but is reported:
        report=False raises MecError(errFileCorrupt) after the healed files were produced (Heal's derr); report=True
        returns (outs, rc, corrupt[n])."""
        files = [None if f is None else _u8(f) for f in files]
        fsz = self.bitrot_file_size(total)
        outs = [np.zeros(fsz, dtype=np.uint8) if stale[i] else None for i in range(self.n)]
        corrupt = np.zeros(self.n, dtype=np.uint8)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        rc = lib().mec_heal_prefer(self.h, _ptrs(files), None if pf is None else pf.ctypes.data, total, _ptrs(outs), corrupt.ctypes.data)
        if report:
            if rc and rc != -7:
                raise MecError(rc, "mec_heal")
            return outs, rc, corrupt
        if rc:
            raise MecError(rc, "mec_heal")
        return outs

    def reconstruct_frames(self, frames, nblocks, last_shard_len, want, data_only=False):
        frames = [None if f is None else _u8(f) for f in frames]
        S = self.shard_size()
        last = last_shard_len or S
        fbytes = (nblocks - 1) * (32 + S) + 32 + last if nblocks else 0
        want = np.asarray(want, dtype=np.uint8)
        outs = [np.zeros(fbytes, dtype=np.uint8) if want[i] else None for i in range(self.n)]
        corrupt = np.zeros(self.n, dtype=np.uint8)
        rc = lib().mec_reconstruct_frames(self.h, _ptrs(frames), nblocks, last_shard_len, want.ctypes.data,
                                          1 if data_only else 0, _ptrs(outs), corrupt.ctypes.data)
        if rc:
            raise MecError(rc, "mec_reconstruct_frames")
        return outs, corrupt

    def bitrot_verify(self, file, part_len):
        f = _u8(file)
        return lib().mec_bitrot_verify(self.h, f.ctypes.data if f.size else None, f.size, part_len)

    def bitrot_verify_batch(self, files, part_lens):
        """mec_bitrot_verify_batch: -> list of 0 / -7 per shard file."""
        files = [_u8(f) for f in files]
        n = len(files)
        fl = (C.c_int64 * n)(*[f.size for f in files])
        pl = (C.c_int64 * n)(*[int(x) for x in part_lens])
        res = (C.c_int32 * n)()
        rc = lib().mec_bitrot_verify_batch(self.h, n, _ptrs(files), fl, pl, res)
        if rc:
            raise MecError(rc, "mec_bitrot_verify_batch")
        return list(res)

    def bitrot_verify_parts(self, files, algos, part_lens, sums=None):
        """mec_bitrot_verify_parts (VerifyFile): part p is files[p] (bytes as stored, None = NULL), written with algos[p], of
        part_lens[p] bytes (streaming parts; ShardFileSize(part.Size)), with the expected whole-file digest sums[p] (bytes or None;
        read for whole-file algorithms only; sums=None passes NULL).  -> list of 0 / -7 / -12 per part."""
        return _verify_parts(lib().mec_bitrot_verify_parts, self.h, "mec_bitrot_verify_parts", files, algos, part_lens, sums)

    # -- legacy whole-file bitrot
    def encode_whole(self, src, online=None, write_quorum=0):
        src = _u8(src)
        flen = self.shard_file_size(src.size)
        online = [True] * self.n if online is None else online
        files = [np.zeros(flen, dtype=np.uint8) if online[i] else None for i in range(self.n)]
        sums = np.zeros((self.n, 64), dtype=np.uint8)
        rc = lib().mec_encode_whole(self.h, src.ctypes.data if src.size else None, src.size, _ptrs(files), sums.ctypes.data, write_quorum)
        if rc < 0:
            raise MecError(rc, "mec_encode_whole")
        ds = lib().mec_digest_size(self.algo)
        return files, [sums[i, :ds].tobytes() for i in range(self.n)]

    def decode_whole(self, files, sums, offset, length, total):
        """Erasure.Decode over wholeBitrotReaders: files = raw shard files (None = offline), sums = their expected digests."""
        files = [None if f is None else _u8(f) for f in files]
        sm = np.zeros((self.n, 64), dtype=np.uint8)
        for i, d in enumerate(sums):
            if d is not None:
                sm[i, :len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
        dst = np.zeros(max(length, 1), dtype=np.uint8)
        hint = C.c_int(0)
        rc = lib().mec_decode_whole(self.h, _ptrs(files), sm.ctypes.data, offset, length, total, dst.ctypes.data, C.byref(hint))
        if rc < 0:
            raise MecError(rc, "mec_decode_whole")
        return dst[:length], hint.value

    def transcode_whole(self, files, sums, total, dst, prefer=None, online=None, write_quorum=0):
        """mec_transcode_whole: move a whole part of `total` bytes written with this codec's whole-file bitrot algorithm — raw shard
        files (None = offline) and their expected digests `sums` — to the geometry of the streaming Codec `dst` without the object
        bytes leaving the device.  online = dst's writers (None = all).  -> (out_files, heal_hint) as Codec.transcode: heal_hint is
        -7 when a reader failed its whole-file digest and the next one took its place."""
        files = [None if f is None else _u8(f) for f in files]
        sm = np.zeros((self.n, 64), dtype=np.uint8)
        for i, d in enumerate(sums):
            if d is not None:
                sm[i, :len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
        fsz = dst.bitrot_file_size(total)
        online = [True] * dst.n if online is None else online
        outs = [np.zeros(fsz, dtype=np.uint8) if online[i] else None for i in range(dst.n)]
        hint = C.c_int(0)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        marker = np.zeros(1, dtype=np.uint8)  # an empty part's online writers still count against the quorum
        optrs = _ptrs([(o if o.size else marker) if o is not None else None for o in outs])
        rc = lib().mec_transcode_whole(self.h, _ptrs(files), sm.ctypes.data, None if pf is None else pf.ctypes.data, total, dst.h,
                                       optrs, write_quorum, C.byref(hint))
        if rc < 0:
            raise MecError(rc, "mec_transcode_whole")
        return outs, hint.value

    def heal_whole(self, files, sums, stale, total):
        """-> (out_files, out_sums, rc, corrupt): rc is 0 or -7 (healed, bitrot met in a source)."""
        files = [None if f is None else _u8(f) for f in files]
        sm = np.zeros((self.n, 64), dtype=np.uint8)
        for i, d in enumerate(sums):
            if d is not None:
                sm[i, :len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
        flen = self.shard_file_size(total)
        outs = [np.zeros(flen, dtype=np.uint8) if stale[i] else None for i in range(self.n)]
        osum = np.zeros((self.n, 64), dtype=np.uint8)
        corrupt = np.zeros(self.n, dtype=np.uint8)
        rc = lib().mec_heal_whole(self.h, _ptrs(files), sm.ctypes.data, total, _ptrs(outs), osum.ctypes.data, corrupt.ctypes.data)
        if rc and rc != -7:
            raise MecError(rc, "mec_heal_whole")
        ds = lib().mec_digest_size(self.algo)
        return outs, [osum[i, :ds].tobytes() if stale[i] else None for i in range(self.n)], rc, corrupt

    def _mixed_args(self, algos, sums):
        al = (C.c_int32 * self.n)(*[int(a) for a in algos])
        if sums is None:
            return al, None
        sm = np.zeros((self.n, 64), dtype=np.uint8)
        for i, d in enumerate(sums):
            if d is not None:
                sm[i, :len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
        return al, sm

    def decode_mixed(self, files, algos, sums, offset, length, total, prefer=None):
        """Erasure.Decode over a part whose drives mix bitrot formats (this codec is HighwayHash256S): algos[i] is drive i's
        algorithm; files[i] its part.N image (HIGHWAYHASH256S) or raw shard file (a whole-file algorithm, expected digest sums[i]);
        None = offline.  sums: list of bytes / None, or None.  -> (bytes, heal_hint) as Codec.decode."""
        files = [None if f is None else _u8(f) for f in files]
        al, sm = self._mixed_args(algos, sums)
        dst = np.zeros(max(length, 1), dtype=np.uint8)
        hint = C.c_int(0)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        rc = lib().mec_decode_mixed(self.h, al, _ptrs(files), None if sm is None else sm.ctypes.data,
                                    None if pf is None else pf.ctypes.data, offset, length, total, dst.ctypes.data, C.byref(hint))
        if rc < 0:
            raise MecError(rc, "mec_decode_mixed")
        return dst[:length], hint.value

    def heal_mixed(self, files, algos, sums, stale, total, prefer=None, report=False):
        """Erasure.Heal as healObject runs it on a part whose drives mix bitrot formats: the stale drives are rebuilt as
        HighwayHash256S part.N images whatever format the readers have (files / algos / sums as decode_mixed; a stale drive is never
        read).  report as Codec.heal."""
        files = [None if f is None else _u8(f) for f in files]
        al, sm = self._mixed_args(algos, sums)
        fsz = self.bitrot_file_size(total)
        outs = [np.zeros(fsz, dtype=np.uint8) if stale[i] else None for i in range(self.n)]
        corrupt = np.zeros(self.n, dtype=np.uint8)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        marker = np.zeros(1, dtype=np.uint8)  # an empty part's stale drives are still marked
        optrs = _ptrs([(o if o.size else marker) if o is not None else None for o in outs])
        rc = lib().mec_heal_mixed(self.h, al, _ptrs(files), None if sm is None else sm.ctypes.data,
                                  None if pf is None else pf.ctypes.data, total, optrs, corrupt.ctypes.data)
        if report:
            if rc and rc != -7:
                raise MecError(rc, "mec_heal_mixed")
            return outs, rc, corrupt
        if rc:
            raise MecError(rc, "mec_heal_mixed")
        return outs

    def whole_hash(self, algo, msgs, msg_len, count):
        msgs = _u8(msgs)
        ds = lib().mec_digest_size(algo)
        out = np.zeros((count, ds), dtype=np.uint8)
        rc = lib().mec_whole_hash(self.h, algo, msgs.ctypes.data if msgs.size else None, msg_len, count, out.ctypes.data)
        if rc:
            raise MecError(rc, "mec_whole_hash")
        return out

    def whole_hash_device(self, algo, d_msgs, pitch, msg_len, count, d_digests, stream=0):
        rc = lib().mec_whole_hash_device(self.h, algo, d_msgs, pitch, msg_len, count, d_digests, stream)
        if rc:
            raise MecError(rc, "mec_whole_hash_device")

    def bitrot_verify_whole(self, algo, file, want):
        f = _u8(file); w = _u8(want)
        return lib().mec_bitrot_verify_whole(self.h, algo, f.ctypes.data if f.size else None, f.size, w.ctypes.data)

    # -- shard shaped
    def rs_encode_shards(self, shards):
        """reedsolomon.Encoder.Encode: list of k+m equally sized arrays, parity written in place."""
        per = shards[0].size
        rc = lib().mec_rs_encode_shards(self.h, _ptrs(shards), per)
        if rc:
            raise MecError(rc, "mec_rs_encode_shards")

    def rs_reconstruct_shards(self, shards, present, data_only=False):
        per = max(s.size for s in shards)
        pres = np.asarray(present, dtype=np.uint8)
        return lib().mec_rs_reconstruct_shards(self.h, _ptrs(shards), pres.ctypes.data, per, 1 if data_only else 0)

    def hh256_batch(self, msgs, msg_len, count):
        msgs = _u8(msgs)
        out = np.zeros((count, 32), dtype=np.uint8)
        rc = lib().mec_hh256_batch(self.h, msgs.ctypes.data if msgs.size else None, msg_len, count, out.ctypes.data)
        if rc:
            raise MecError(rc, "mec_hh256_batch")
        return out

    def encode_data(self, data):
        """Erasure.EncodeData (cmd/erasure-coding.go:77): Split + Encode -> k+m shard arrays."""
        data = _u8(data)
        if data.size == 0:
            return [np.zeros(0, dtype=np.uint8) for _ in range(self.n)]
        per = -(-data.size // self.k)
        store = np.zeros(self.n * per, dtype=np.uint8)
        store[:data.size] = data
        shards = [store[i * per:(i + 1) * per] for i in range(self.n)]
        if self.m:
            self.rs_encode_shards(shards)
        return shards


class Batcher:
    """mec_batcher: concurrent PutObject calls of one geometry merged into shared launches.  encode() may be called from many
    threads at once (ctypes releases the GIL for the duration of the call).  mix_patterns=True (MEC_BATCHER_MIX_PATTERNS): GETs
    and heals of different erasure patterns (reader sets, stale sets) share batches.  dst=(k2, m2) (mec_batcher_new_transcode): the
    batcher also moves parts of its geometry to RS(k2, m2) of the same block size (transcode()); dst=(k2, m2, dst_block_size)
    (mec_batcher_new_transcode_ex): to RS(k2, m2) with a block size that divides block_size (legacy 10 MiB parts into 1 MiB)."""

    def __init__(self, k, m, block_size=1 << 20, device=0, max_batch_blocks=256, max_wait_us=200, mix_patterns=False, dst=None):
        h = C.c_void_p()
        flags = MIX_PATTERNS if mix_patterns else 0
        if dst is None:
            rc = lib().mec_batcher_new_ex(k, m, block_size, device, max_batch_blocks, max_wait_us, flags, C.byref(h))
        elif len(dst) == 2:
            rc = lib().mec_batcher_new_transcode(k, m, dst[0], dst[1], block_size, device, max_batch_blocks, max_wait_us, flags,
                                                 C.byref(h))
        else:
            rc = lib().mec_batcher_new_transcode_ex(k, m, block_size, dst[0], dst[1], dst[2], device, max_batch_blocks, max_wait_us,
                                                    flags, C.byref(h))
        if rc:
            raise MecError(rc, "mec_batcher_new_ex" if dst is None else "mec_batcher_new_transcode")
        self.h, self.k, self.m, self.n, self.block_size = h, k, m, k + m, block_size
        self._sizes = Codec(k, m, block_size, device=device)
        self._dst_sizes = None if dst is None else Codec(dst[0], dst[1], dst[2] if len(dst) > 2 else block_size, device=device)

    def _encode_crc(self, src, files, dd, write_quorum, checksums):
        """mec_batcher_encode_crc -> (CRC32, CRC32C, CRC64NVME), 0 where not asked for"""
        out = (C.c_uint64 * 3)()
        rc = lib().mec_batcher_encode_crc(self.h, src.ctypes.data if src.size else None, src.size, _ptrs(files),
                                          None if dd is None else dd.ctypes.data, write_quorum, checksums, out)
        if rc < 0:
            raise MecError(rc, "mec_batcher_encode_crc")
        return tuple(int(v) for v in out)

    def _encode_sums(self, src, files, dd, write_quorum, checksums, hashes):
        """mec_batcher_encode_sums -> ((CRC32, CRC32C, CRC64NVME), {"md5": ..., "sha1": ..., "sha256": ...} for the bits of hashes)"""
        out = (C.c_uint64 * 3)()
        rec = (C.c_uint8 * SUM_BYTES)()
        rc = lib().mec_batcher_encode_sums(self.h, src.ctypes.data if src.size else None, src.size, _ptrs(files),
                                           None if dd is None else dd.ctypes.data, write_quorum, checksums | hashes, out, rec)
        if rc < 0:
            raise MecError(rc, "mec_batcher_encode_sums")
        return tuple(int(v) for v in out), {name: bytes(rec[o:o + n]) for name, (bit, o, n) in SUM_SLOTS.items() if hashes & bit}

    def encode(self, src, online=None, write_quorum=0, pinned=False, checksums=0, hashes=0):
        """pinned=True: the part files are allocated page-locked (and `src` must be, e.g. a pinned_array) — the batch then moves
        through the gather / scatter kernels instead of per-request copies.  The caller owns (and should free) those arrays.
        checksums: a mask of CRC32 / CRC32C / CRC64NVME; non-zero returns (files, (crc32, crc32c, crc64nvme)) computed on the
        bytes the batch staged (mec_batcher_encode_crc).  hashes: a mask of SUM_MD5 / SUM_SHA1 / SUM_SHA256; non-zero appends
        {"md5": bytes, "sha1": bytes, "sha256": bytes} with the keys asked for (mec_batcher_encode_sums)."""
        src = _u8(src)
        fsz = self._sizes.bitrot_file_size(src.size)
        online = [True] * self.n if online is None else online
        mk = (lambda nb: pinned_array(max(nb, 1))[:nb]) if pinned else (lambda nb: np.zeros(nb, dtype=np.uint8))
        files = [mk(fsz) if online[i] else None for i in range(self.n)]
        if hashes:
            crcs, sums = self._encode_sums(src, files, None, write_quorum, checksums, hashes)
            return (files, crcs, sums) if checksums else (files, sums)
        if checksums:
            return files, self._encode_crc(src, files, None, write_quorum, checksums)
        rc = lib().mec_batcher_encode(self.h, src.ctypes.data if src.size else None, src.size, _ptrs(files), write_quorum)
        if rc < 0:
            raise MecError(rc, "mec_batcher_encode")
        return files

    def encode_sg(self, src, online=None, write_quorum=0, pinned=False, checksums=0, hashes=0):
        """mec_batcher_encode_sg: -> (files, data_digests) shaped like Codec.encode_sg.  pinned=True: the parity images and the
        [block][k][32] digest array are page-locked (and `src` must be), so the scatter kernel writes both; the caller owns them.
        checksums: as for encode(); non-zero returns (files, data_digests, (crc32, crc32c, crc64nvme)).  hashes: as for encode();
        non-zero appends the digest dict."""
        src = _u8(src)
        fsz = self._sizes.bitrot_file_size(src.size)
        nb = -(-src.size // self.block_size)
        online = [True] * self.n if online is None else online
        mk = (lambda nb: pinned_array(max(nb, 1))[:nb]) if pinned else (lambda nb: np.zeros(nb, dtype=np.uint8))
        marker = np.zeros(1, dtype=np.uint8)  # data drives: only NULL / non-NULL is looked at
        files = [(mk(fsz) if i >= self.k else marker) if online[i] else None for i in range(self.n)]
        dd = mk(max(nb, 1) * self.k * 32).reshape(max(nb, 1), self.k, 32)
        if hashes:
            crcs, sums = self._encode_sums(src, files, dd, write_quorum, checksums, hashes)
            files = [f if i >= self.k else None for i, f in enumerate(files)]
            return (files, dd[:nb], crcs, sums) if checksums else (files, dd[:nb], sums)
        if checksums:
            crcs = self._encode_crc(src, files, dd, write_quorum, checksums)
            return [f if i >= self.k else None for i, f in enumerate(files)], dd[:nb], crcs
        rc = lib().mec_batcher_encode_sg(self.h, src.ctypes.data if src.size else None, src.size, _ptrs(files), dd.ctypes.data,
                                         write_quorum)
        if rc < 0:
            raise MecError(rc, "mec_batcher_encode_sg")
        return [f if i >= self.k else None for i, f in enumerate(files)], dd[:nb]

    def decode(self, files, offset, length, total, dst=None, prefer=None):
        """mec_batcher_decode_prefer: files = part-file arrays (None = offline); pass page-locked arrays (and a page-locked dst) to
        ride in merged launches.  prefer = n flags (preferReaders), None = mec_batcher_decode.  -> (bytes, heal_hint)"""
        files = [None if f is None else _u8(f) for f in files]
        if dst is None:
            dst = np.zeros(max(length, 1), dtype=np.uint8)
        hint = C.c_int(0)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        rc = lib().mec_batcher_decode_prefer(self.h, _ptrs(files), None if pf is None else pf.ctypes.data, offset, length, total,
                                             dst.ctypes.data, C.byref(hint))
        if rc < 0:
            raise MecError(rc, "mec_batcher_decode_prefer")
        return dst[:length], hint.value

    def heal(self, files, stale, total, prefer=None, pinned=False):
        """mec_batcher_heal: -> (outs, rc, corrupt[n]) like Codec.heal(report=True).  Page-locked part files and pinned=True (the out
        files are allocated page-locked; the caller owns and should free them) let the heal ride in merged launches."""
        files = [None if f is None else _u8(f) for f in files]
        fsz = self._sizes.bitrot_file_size(total)
        mk = (lambda nb: pinned_array(max(nb, 1))[:nb]) if pinned else (lambda nb: np.zeros(nb, dtype=np.uint8))
        outs = [mk(fsz) if stale[i] else None for i in range(self.n)]
        corrupt = np.zeros(self.n, dtype=np.uint8)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        rc = lib().mec_batcher_heal(self.h, _ptrs(files), None if pf is None else pf.ctypes.data, total, _ptrs(outs), corrupt.ctypes.data)
        if rc and rc != -7:
            raise MecError(rc, "mec_batcher_heal")
        return outs, rc, corrupt

    def transcode(self, files, total, prefer=None, online=None, write_quorum=0, pinned=False):
        """mec_batcher_transcode (a batcher made with dst=): move a whole part of `total` bytes from this geometry's part files (None
        = offline) to the destination geometry.  online = the destination's writers (None = all).  Page-locked part files and
        pinned=True (the out files are allocated page-locked; the caller owns and should free them) let the move ride in merged
        batches.  -> (out_files, heal_hint) as Codec.transcode."""
        if self._dst_sizes is None:
            raise MecError(-12, "mec_batcher_transcode")
        files = [None if f is None else _u8(f) for f in files]
        n2 = self._dst_sizes.n
        fsz = self._dst_sizes.bitrot_file_size(total)
        online = [True] * n2 if online is None else online
        mk = (lambda nb: pinned_array(max(nb, 1))[:nb]) if pinned else (lambda nb: np.zeros(nb, dtype=np.uint8))
        outs = [mk(fsz) if online[i] else None for i in range(n2)]
        hint = C.c_int(0)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        # an empty part has empty out files, yet an online writer must still count against the quorum
        marker = np.zeros(1, dtype=np.uint8)
        optrs = _ptrs([(o if o.size else marker) if o is not None else None for o in outs])
        rc = lib().mec_batcher_transcode(self.h, _ptrs(files), None if pf is None else pf.ctypes.data, total, optrs, write_quorum,
                                         C.byref(hint))
        if rc < 0:
            raise MecError(rc, "mec_batcher_transcode")
        return outs, hint.value

    def transcode_whole(self, files, sums, total, algo, prefer=None, online=None, write_quorum=0, pinned=False):
        """mec_batcher_transcode_whole (a batcher made with dst=): move a whole part of `total` bytes written with the whole-file
        bitrot algorithm `algo` (SHA256, BLAKE2B512 or HIGHWAYHASH256) — raw shard files (None = offline) and their expected digests
        `sums` — to the destination geometry.  online / write_quorum / pinned as transcode(): page-locked shard files and pinned=True
        let the move ride in merged batches.  -> (out_files, heal_hint) as Codec.transcode_whole."""
        files = [None if f is None else _u8(f) for f in files]
        sm = np.zeros((self.n, 64), dtype=np.uint8)
        for i, d in enumerate(sums):
            if d is not None:
                sm[i, :len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
        n2 = self._dst_sizes.n if self._dst_sizes is not None else 0
        fsz = self._dst_sizes.bitrot_file_size(total) if self._dst_sizes is not None else 0
        online = [True] * n2 if online is None else online
        mk = (lambda nb: pinned_array(max(nb, 1))[:nb]) if pinned else (lambda nb: np.zeros(nb, dtype=np.uint8))
        outs = [mk(fsz) if online[i] else None for i in range(n2)]
        hint = C.c_int(0)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        marker = np.zeros(1, dtype=np.uint8)  # an empty part's online writers still count against the quorum
        optrs = _ptrs([(o if o.size else marker) if o is not None else None for o in outs]) if n2 else (C.c_void_p * 1)()
        rc = lib().mec_batcher_transcode_whole(self.h, algo, _ptrs(files), sm.ctypes.data, None if pf is None else pf.ctypes.data,
                                               total, optrs, write_quorum, C.byref(hint))
        if rc < 0:
            raise MecError(rc, "mec_batcher_transcode_whole")
        return outs, hint.value

    def decode_mixed(self, files, algos, sums, offset, length, total, dst=None, prefer=None):
        """mec_batcher_decode_mixed: Codec.decode_mixed through the coalescer (files / algos / sums / prefer as there; page-locked
        readers and a page-locked dst let the call ride in merged batches).  -> (bytes, heal_hint)"""
        files = [None if f is None else _u8(f) for f in files]
        al, sm = self._sizes._mixed_args(algos, sums)
        if dst is None:
            dst = np.zeros(max(length, 1), dtype=np.uint8)
        hint = C.c_int(0)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        rc = lib().mec_batcher_decode_mixed(self.h, al, _ptrs(files), None if sm is None else sm.ctypes.data,
                                            None if pf is None else pf.ctypes.data, offset, length, total, dst.ctypes.data,
                                            C.byref(hint))
        if rc < 0:
            raise MecError(rc, "mec_batcher_decode_mixed")
        return dst[:length], hint.value

    def heal_mixed(self, files, algos, sums, stale, total, prefer=None, report=False, pinned=False):
        """mec_batcher_heal_mixed: Codec.heal_mixed through the coalescer (arguments, report and results as there).  Page-locked
        readers and pinned=True (the out files are allocated page-locked; the caller owns and should free them) let the heal ride
        in merged batches."""
        files = [None if f is None else _u8(f) for f in files]
        al, sm = self._sizes._mixed_args(algos, sums)
        fsz = self._sizes.bitrot_file_size(total)
        mk = (lambda nb: pinned_array(max(nb, 1))[:nb]) if pinned else (lambda nb: np.zeros(nb, dtype=np.uint8))
        outs = [mk(fsz) if stale[i] else None for i in range(self.n)]
        corrupt = np.zeros(self.n, dtype=np.uint8)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        marker = np.zeros(1, dtype=np.uint8)  # an empty part's stale drives are still marked
        optrs = _ptrs([(o if o.size else marker) if o is not None else None for o in outs])
        rc = lib().mec_batcher_heal_mixed(self.h, al, _ptrs(files), None if sm is None else sm.ctypes.data,
                                          None if pf is None else pf.ctypes.data, total, optrs, corrupt.ctypes.data)
        if report:
            if rc and rc != -7:
                raise MecError(rc, "mec_batcher_heal_mixed")
            return outs, rc, corrupt
        if rc:
            raise MecError(rc, "mec_batcher_heal_mixed")
        return outs

    def verify(self, files, algos, part_lens, sums=None):
        """mec_batcher_verify: Codec.bitrot_verify_parts through the coalescer on this batcher's geometry (arguments and results as
        there).  Page-locked files (pinned_array) let the call ride in merged batches."""
        return _verify_parts(lib().mec_batcher_verify, self.h, "mec_batcher_verify", files, algos, part_lens, sums)

    def encode_sse(self, src, key, nonce, online=None, write_quorum=0, pinned=False):
        """mec_batcher_encode_sse: Codec.encode_sse through the coalescer -> part files.  A page-locked `src` (pinned_array) and
        pinned=True (the part files are allocated page-locked; the caller owns and should free them) let the call ride in merged
        batches."""
        src, key, nonce = _u8(src), _u8(key), _u8(nonce)
        if key.size != 32 or nonce.size != 12:
            raise ValueError("key is 32 bytes, nonce 12")
        fsz = self._sizes.bitrot_file_size(dare_encrypted_size(src.size))
        online = [True] * self.n if online is None else online
        mk = (lambda nb: pinned_array(max(nb, 1))[:nb]) if pinned else (lambda nb: np.zeros(nb, dtype=np.uint8))
        files = [mk(fsz) if online[i] else None for i in range(self.n)]
        rc = lib().mec_batcher_encode_sse(self.h, src.ctypes.data if src.size else None, src.size, key.ctypes.data, nonce.ctypes.data,
                                          _ptrs(files), write_quorum)
        if rc < 0:
            raise MecError(rc, "mec_batcher_encode_sse")
        return files

    def decode_sse(self, files, offset, length, enc_total, key, prefer=None, dst=None):
        """mec_batcher_decode_sse: Codec.decode_sse through the coalescer; page-locked part files and a page-locked dst let the
        call ride in merged batches.  -> (plaintext [offset, offset + length), heal_hint)"""
        files = [None if f is None else _u8(f) for f in files]
        key = _u8(key)
        if key.size != 32:
            raise ValueError("key is 32 bytes")
        if dst is None:
            dst = np.zeros(max(length, 1), dtype=np.uint8)
        hint = C.c_int(0)
        pf = None if prefer is None else np.asarray(prefer, dtype=np.uint8)
        rc = lib().mec_batcher_decode_sse(self.h, _ptrs(files), None if pf is None else pf.ctypes.data, offset, length, enc_total,
                                          key.ctypes.data, dst.ctypes.data, C.byref(hint))
        if rc < 0:
            raise MecError(rc, "mec_batcher_decode_sse")
        return dst[:length], hint.value

    def set_option(self, name, value):
        """mec_batcher_set_option: "dare_chacha20" (0, 1, 2) for requests admitted from now on"""
        rc = lib().mec_batcher_set_option(self.h, name.encode(), int(value))
        if rc:
            raise MecError(rc, "mec_batcher_set_option")

    def stat(self, name):
        return lib().mec_batcher_stat(self.h, name.encode())

    def close(self):
        if getattr(self, "h", None):
            lib().mec_batcher_free(self.h)
            self.h = None
            self._sizes.close()
            if self._dst_sizes is not None:
                self._dst_sizes.close()

    __del__ = close


def dare_encrypted_size(n):
    """sio.EncryptedSize; MecError on an invalid size"""
    v = lib().mec_dare_encrypted_size(n)
    if v < 0:
        raise MecError(v, "mec_dare_encrypted_size")
    return v


def dare_decrypted_size(n):
    """sio.DecryptedSize; MecError on an invalid size"""
    v = lib().mec_dare_decrypted_size(n)
    if v < 0:
        raise MecError(v, "mec_dare_decrypted_size")
    return v


def pinned_array(nbytes, device=None):
    """uint8 numpy array over page-locked host memory from mec_alloc_pinned (bpool.BytePoolCap's role) — with `device`, on the
    NUMA node of that GPU (mec_alloc_pinned_on); never freed by the array — keep it for the life of the process or release
    it with lib().mec_free_pinned(arr.ctypes.data)."""
    p = lib().mec_alloc_pinned(max(int(nbytes), 1)) if device is None else lib().mec_alloc_pinned_on(int(device), max(int(nbytes), 1))
    if not p:
        raise MecError(-100, "mec_alloc_pinned")
    return np.ctypeslib.as_array((C.c_uint8 * int(nbytes)).from_address(p))


def heal_batch(pool, objects, outs=None):
    """mec_heal_batch: `pool` = list of Codec handles of one geometry, `objects` = list of (files, stale, total).
    Returns the rebuilt shard files per object (None where not stale).  `outs` = preallocated output arrays per object
    (e.g. pinned_array of bitrot_file_size(total) bytes where stale, None elsewhere); default: fresh pageable arrays."""
    n = pool[0].n
    handles = (C.c_void_p * len(pool))(*[c.h for c in pool])
    keep, fptrs, optrs, outs_all = [], [], [], []
    for o, (files, stale, total) in enumerate(objects):
        files = [None if f is None else _u8(f) for f in files]
        fsz = pool[0].bitrot_file_size(total)
        obj_outs = outs[o] if outs is not None else [np.zeros(fsz, dtype=np.uint8) if stale[i] else None for i in range(n)]
        fp, op = _ptrs(files), _ptrs(obj_outs)
        keep += [files, fp, op]
        fptrs.append(C.cast(fp, C.c_void_p)); optrs.append(C.cast(op, C.c_void_p)); outs_all.append(obj_outs)
    nobj = len(objects)
    fa = (C.c_void_p * nobj)(*fptrs); oa = (C.c_void_p * nobj)(*optrs)
    totals = (C.c_int64 * nobj)(*[t for _, _, t in objects])
    rcs = (C.c_int32 * nobj)()
    rc = lib().mec_heal_batch(handles, len(pool), nobj, fa, totals, oa, rcs)
    if rc:
        raise MecError(rc, "mec_heal_batch")
    return outs_all
