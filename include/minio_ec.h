/*
 * minio_ec.h — C ABI of the H100 erasure-code + bitrot library (libminio_ec.so).
 *
 * Drop-in boundary for MinIO's erasure hot path.  The reference has no FFI here — the path sits
 * behind Go interfaces (reedsolomon.Encoder held by `Erasure.encoder`, hash.Hash from
 * BitrotAlgorithm.New, io.Writer / io.ReaderAt per drive).  Each entry point names the reference
 * function whose body a cgo binding would replace (file:line under /root/reference); the Go-side
 * stub is written out in INTEGRATION.md.  Plain pointers and sizes only; no retained caller memory.
 *
 * Return codes: 0 / non-negative = success, negative = one of MEC_ERR_*.
 */
#ifndef MINIO_EC_H
#define MINIO_EC_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- errors: reedsolomon.Err* (go.mod:49) and MinIO storage errors ------------------------- */
enum {
  MEC_OK = 0,
  MEC_ERR_INV_SHARD_NUM = -1,     /* reedsolomon.ErrInvShardNum   cmd/erasure-coding.go:45 */
  MEC_ERR_MAX_SHARD_NUM = -2,     /* reedsolomon.ErrMaxShardNum   cmd/erasure-coding.go:49 */
  MEC_ERR_TOO_FEW_SHARDS = -3,    /* reedsolomon.ErrTooFewShards */
  MEC_ERR_SHARD_NO_DATA = -4,     /* reedsolomon.ErrShardNoData */
  MEC_ERR_SHARD_SIZE = -5,        /* reedsolomon.ErrShardSize */
  MEC_ERR_SHORT_DATA = -6,        /* reedsolomon.ErrShortData */
  MEC_ERR_FILE_CORRUPT = -7,      /* errFileCorrupt        cmd/storage-errors.go:104 */
  MEC_ERR_LESS_DATA = -8,         /* errLessData           cmd/storage-errors.go:114 */
  MEC_ERR_UNEXPECTED = -9,        /* errUnexpected         cmd/storage-errors.go:29 */
  MEC_ERR_READ_QUORUM = -10,      /* errErasureReadQuorum  cmd/erasure-errors.go:23 */
  MEC_ERR_WRITE_QUORUM = -11,     /* errErasureWriteQuorum cmd/erasure-errors.go:26 */
  MEC_ERR_INVALID_ARGUMENT = -12, /* errInvalidArgument */
  MEC_ERR_NOT_AUTHENTIC = -13,    /* sio.NotAuthentic -> errObjectTampered  cmd/encryption-v1.go:57 */
  MEC_ERR_SIGNATURE_MISMATCH = -14, /* errSignatureMismatch  cmd/typed-errors.go:31 */
  MEC_ERR_MALFORMED_ENCODING = -15, /* errMalformedEncoding  cmd/streaming-signature-v4.go:184 */
  MEC_ERR_CHUNK_TOO_BIG = -16,      /* errChunkTooBig        cmd/streaming-signature-v4.go:187 */
  MEC_ERR_INCOMPLETE_BODY = -17,    /* io.ErrUnexpectedEOF / IncompleteBody  cmd/erasure-object.go:1450-1453 */
  MEC_ERR_OVERREAD = -18,           /* ioutil.ErrOverread    internal/ioutil/hardlimitreader.go:27 */
  MEC_ERR_CUDA = -100,            /* CUDA runtime / driver failure (see mec_last_error) */
  MEC_ERR_NO_DEVICE = -101,       /* no CUDA device: the library never falls back to the CPU */
  MEC_ERR_UNSUPPORTED = -102      /* geometry or algorithm outside the GPU path (see DESIGN.md) */
};

/* ---- bitrot algorithms: cmd/xl-storage-format-v1.go:142-159 -------------------------------- */
enum { MEC_SHA256 = 1, MEC_HIGHWAYHASH256 = 2, MEC_HIGHWAYHASH256S = 3, MEC_BLAKE2B512 = 4 };

typedef struct mec_codec mec_codec;

/* ---- lifecycle ----------------------------------------------------------------------------- */
/* NewErasure (cmd/erasure-coding.go:42): validates k>0, m>=0, k+m<=256 with the same errors.
 * `device` is the CUDA ordinal.  One codec may be shared by threads; calls serialise per codec. */
int mec_codec_new(int k, int m, int64_t block_size, int bitrot_algo, int device, mec_codec** out);
void mec_codec_free(mec_codec* c);
int mec_device_count(void);
const char* mec_last_error(void); /* thread-local description of the last MEC_ERR_CUDA */
const char* mec_version(void);

/* ---- size helpers -------------------------------------------------------------------------- */
int64_t mec_shard_size(const mec_codec* c);                                  /* Erasure.ShardSize       cmd/erasure-coding.go:116 */
int64_t mec_shard_file_size(const mec_codec* c, int64_t total_length);       /* Erasure.ShardFileSize   cmd/erasure-coding.go:121 */
int64_t mec_shard_file_offset(const mec_codec* c, int64_t start_offset, int64_t length,
                              int64_t total_length);                         /* Erasure.ShardFileOffset cmd/erasure-coding.go:135 */
int64_t mec_bitrot_shard_file_size(int64_t size, int64_t shard_size, int algo); /* bitrotShardFileSize cmd/bitrot.go:156 */
int64_t mec_ceil_frac(int64_t numerator, int64_t denominator);               /* ceilFrac cmd/utils.go:689 */

/* ---- pinned host memory for the byte pool (internal/bpool/bpool.go:25-93; AllocAligned :52,68) ------
 * mec_alloc_pinned: page-locked memory, wherever the calling thread runs.  mec_alloc_pinned_on: page-locked memory on the
 * NUMA node of CUDA device `device` (/sys/bus/pci/devices/<bdf>/numa_node; mbind + first touch + cudaHostRegister) — on a
 * multi-socket box every GPU should stream from the memory behind its own root port.  Both are released with
 * mec_free_pinned.  mec_device_numa_node returns that node (-1 unknown); mec_bind_thread_to_device restricts the calling
 * thread to the CPUs of that node (never beyond its current affinity mask) and returns the node, or -1 when it could not.
 * mec_is_pinned: 1 when `p` is page-locked memory known to CUDA (the host-buffer entry points DMA straight from / into it). */
void* mec_alloc_pinned(size_t bytes);
void* mec_alloc_pinned_on(int device, size_t bytes);
void mec_free_pinned(void* p);
int mec_device_numa_node(int device);
int mec_bind_thread_to_device(int device);
int mec_is_pinned(const void* p);

/* ---- fused block encode: the body of Erasure.EncodeData (cmd/erasure-coding.go:77-91) plus
 * the HighwayHash256 of every shard that streamingBitrotWriter.Write computes
 * (cmd/bitrot-streaming.go:57-59), for ALL erasure blocks of `src` in one call.
 *   src      : len object bytes (host).  Blocks are block_size bytes; the last may be short.
 *   parity   : receives parity shard j of block b at parity + (b*m + j)*shard_size  (host)
 *   digests  : receives 32-byte digest of shard i of block b at digests + (b*(k+m)+i)*32 (host)
 * Data shards alias `src` exactly as Split does (shard i of block b = src[b*block_size + i*S_b ..),
 * zero padded), so they are not copied back.  len == 0 is a no-op (EncodeData returns nil shards). */
int mec_encode_blocks(mec_codec* c, const uint8_t* src, int64_t len, uint8_t* parity, uint8_t* digests);

/* Same, device-resident: d_src/d_parity/d_digests are device pointers on the codec's device,
 * d_src 16-byte aligned, parity row pitch `parity_pitch` (multiple of 16, >= shard_size):
 * parity shard (b, j) at d_parity + (b*m + j)*parity_pitch.  Asynchronous on `cuda_stream`
 * (a cudaStream_t, may be NULL).  d_digests == NULL computes parity only (whole-file bitrot algorithms). */
int mec_encode_blocks_device(mec_codec* c, const uint8_t* d_src, int64_t len, uint8_t* d_parity,
                             int64_t parity_pitch, uint8_t* d_digests, void* cuda_stream);

/* ---- fused block reconstruct: Erasure.DecodeDataBlocks / DecodeDataAndParityBlocks
 * (cmd/erasure-coding.go:94-113 -> reedsolomon ReconstructData / Reconstruct) fused with the
 * digest check of streamingBitrotReader.ReadAt (cmd/bitrot-streaming.go:186-196).
 *   frames[i]   : host pointer to shard file i in streaming-bitrot layout ([32B digest][shard])*,
 *                 or NULL when the drive is offline.  All `nblocks` blocks are full blocks except
 *                 that the last block's shard length is `last_shard_len` (0 => shard_size; a value
 *                 below 0 or above shard_size is MEC_ERR_INVALID_ARGUMENT, checked before any device work).
 *   want[i]     : 1 = out[i] receives shard file i (same frame layout): copied from frames[i] when
 *                 file i is one of the readers, otherwise rebuilt with recomputed digests
 *   data_only   : ReconstructData semantics (parity never rebuilt: out[i] of a wanted parity shard
 *                 that is not read is left as it was)
 *   corrupt[i]  : (optional, n bytes, cleared on entry) set to 1 when a frame of file i that was read
 *                 fails its digest.  Only the files read are checked; the others are never looked at.
 * The first k readable files in index order are read (parallelReader.Read, cmd/erasure-decode.go:127).
 * A reader whose frame fails its digest is dropped for the rest of the call: the blocks before that
 * frame stand, and the call resumes at it with the next readable file.  A wanted reader that is
 * dropped is passed through up to the bad frame and, unless it is parity under data_only, rebuilt
 * from there.  When the readable files run out (initially, or after drops) the call returns
 * MEC_ERR_READ_QUORUM; corrupt[] then names every reader it dropped, so a caller that handed over
 * only k files can drop those and call again with the next ones (include/minio_erasure.hpp,
 * readAndReconstruct).  The out[] files are complete only when the call returns MEC_OK. */
int mec_reconstruct_frames(mec_codec* c, const uint8_t* const* frames, int64_t nblocks,
                           int64_t last_shard_len, const uint8_t* want, int data_only,
                           uint8_t* const* out, uint8_t* corrupt);

/* Device-resident variant of the fused reconstruct (BASELINE configs 3 and 4): d_frames[i] is a device
 * pointer to shard file i in frame layout with a 16-byte aligned `frame_pitch` (>= 32 + shard_size;
 * digest at +0, shard bytes at +32 of every frame), or NULL when the shard is unavailable.  The first k
 * non-NULL files are read; every shard with want[i] != 0 that was not read is rebuilt into
 * d_out + (b*r + q)*out_pitch (q = rank of i among the rebuilt shards) and its digest written to
 * d_digests[(b*(k+r) + k + q)*32]; digests of the k shards read land in d_digests[(b*(k+r) + t)*32] and
 * d_corrupt[b*k + t] is set when frame t of block b fails its stored digest.  All nblocks are full blocks.
 * `flags`: MEC_RECONSTRUCT_DATA_ONLY = ReconstructData semantics (parity never rebuilt);
 * MEC_RECONSTRUCT_NO_OUTPUT_DIGESTS = the rebuilt shards are not hashed (GetObject consumes their bytes only,
 * cmd/erasure-decode.go:283-289; the k shards read are still hashed and checked), their digest slots stay untouched.
 * d_corrupt != NULL requires d_digests != NULL (the digest check runs in the hash threads; MEC_ERR_INVALID_ARGUMENT otherwise);
 * with d_digests == NULL nothing is hashed or verified.
 * Asynchronous on `cuda_stream`; the fail-over policy stays with the caller (see mec_reconstruct_frames). */
#define MEC_RECONSTRUCT_DATA_ONLY 1
#define MEC_RECONSTRUCT_NO_OUTPUT_DIGESTS 2
int mec_reconstruct_device(mec_codec* c, const uint8_t* const* d_frames, int64_t frame_pitch, int64_t nblocks,
                           const uint8_t* want, int flags, uint8_t* d_out, int64_t out_pitch,
                           uint8_t* d_digests, uint8_t* d_corrupt, void* cuda_stream);

/* ---- whole-part drivers ------------------------------------------------------------------- */
/* Erasure.Encode (cmd/erasure-encode.go:69) with one streaming bitrot writer per shard
 * (cmd/bitrot.go:105, cmd/bitrot-streaming.go:44): files[i] (host, or NULL = offline writer)
 * receives exactly the bytes of part.N on drive i; each must hold
 * mec_bitrot_shard_file_size(mec_shard_file_size(len)) bytes.  Fails with MEC_ERR_WRITE_QUORUM
 * when fewer than `write_quorum` writers are online.  Returns bytes consumed. */
int64_t mec_encode(mec_codec* c, const uint8_t* src, int64_t len, uint8_t* const* files, int write_quorum);
/* The same call in the shape streamingBitrotWriter.Write actually has (cmd/bitrot-streaming.go:57-69: w.Write(hash), then
 * w.Write(p) — the shard bytes are never copied next to their digest): the k data shards stay inside `src`, where Split
 * aliased them (cmd/erasure-coding.go:81), and only what the GPU produced comes back —
 *   files[k..n)   : complete part.N images of the parity drives (NULL = offline), written by DMA straight from device memory
 *   data_digests  : digest of data shard i of block b at data_digests + (b*k + i)*32; writer i emits, per block,
 *                   {data_digests[b][i], src + b*block_size + i*S_b (zero padded to S_b)}  (writev / the cgo writeHashed stub)
 *   files[0..k)   : only tested for NULL (offline writers count against write_quorum)
 * No assembly copy exists anywhere on this path.  Returns bytes consumed. */
int64_t mec_encode_sg(mec_codec* c, const uint8_t* src, int64_t len, uint8_t* const* files, uint8_t* data_digests,
                      int write_quorum);

/* Erasure.Decode (cmd/erasure-decode.go:239) over streaming bitrot readers: writes object bytes
 * [offset, offset+length) of a part of `total_length` bytes to dst.  files[i] NULL = offline.
 * Returns bytes written; *heal_hint is set to MEC_ERR_FILE_CORRUPT when a frame failed its digest
 * but the read still succeeded (the errFileCorrupt side-band of cmd/erasure-decode.go:288-293). */
int64_t mec_decode(mec_codec* c, const uint8_t* const* files, int64_t offset, int64_t length,
                   int64_t total_length, uint8_t* dst, int* heal_hint);

/* Same with parallelReader.preferReaders (cmd/erasure-decode.go:92-123; `prefer` as passed by
 * cmd/erasure-object.go:387 for local drives): readers with prefer[i] != 0 are tried before the others, each
 * class in index order.  prefer == NULL is mec_decode. */
int64_t mec_decode_prefer(mec_codec* c, const uint8_t* const* files, const uint8_t* prefer, int64_t offset,
                          int64_t length, int64_t total_length, uint8_t* dst, int* heal_hint);

/* Erasure.Heal (cmd/erasure-decode.go:317): rebuilds every shard file with out_files[i] != NULL
 * from the readable files (NULL = offline / stale). */
int mec_heal(mec_codec* c, const uint8_t* const* files, int64_t total_length, uint8_t* const* out_files);
/* Heal with its `prefer` argument and the bitrot side-band.  Returns MEC_OK, or MEC_ERR_FILE_CORRUPT when the stale shards
 * WERE rebuilt and written but a source reader failed its digest on the way — Heal's derr (cmd/erasure-decode.go:338-341,366;
 * healObject aborts the part on it, cmd/erasure-healing.go:603-608); corrupt[i] (optional, n bytes) names those readers.
 * mec_heal is this call with prefer = NULL, corrupt = NULL and returns the same codes. */
int mec_heal_prefer(mec_codec* c, const uint8_t* const* files, const uint8_t* prefer, int64_t total_length,
                    uint8_t* const* out_files, uint8_t* corrupt);
/* Heal of many objects (BASELINE config 4; healObject fan-out of cmd/global-heal.go:152): object o has files[o][0..n),
 * totals[o], out_files[o][0..n) with mec_heal's meaning.  `pool` holds npool codec handles of the same geometry (each owns
 * its streams and staging buffers); one host thread per handle pulls objects, so staging, kernels and copy-back of
 * different objects overlap.  rcs (optional) receives the per-object result (MEC_ERR_FILE_CORRUPT = healed, a source reader
 * failed its digest); the return value is the first result that is neither MEC_OK nor MEC_ERR_FILE_CORRUPT. */
int mec_heal_batch(mec_codec* const* pool, int npool, int64_t nobjects, const uint8_t* const* const* files,
                   const int64_t* total_lengths, uint8_t* const* const* out_files, int* rcs);

/* Data movement between pools (decommissionObject / rebalanceObject, cmd/erasure-server-pool-decom.go:605,
 * cmd/erasure-server-pool-rebalance.go:848): Erasure.Decode of a whole part on `src` followed by Erasure.Encode of the same
 * bytes on `dst`, without the object leaving the device.  files / prefer / total_length as mec_decode_prefer (whole part,
 * offset 0): the first k readable files are read, preferred ones first, and a reader whose frame fails its digest is dropped for
 * the rest of the call, the part resuming at that block with the next reader.  out_files / write_quorum as mec_encode (complete
 * part.N images of dst's geometry, NULL = offline writer).  Returns total_length, or a negative MEC_ERR_*; *heal_hint =
 * MEC_ERR_FILE_CORRUPT when a source frame failed its digest but the part was still moved.
 * dst's block size may be src's or a whole fraction of it: src block_size = R x dst block_size for an integer R >= 1 (a legacy
 * part written with blockSizeV1 = 10 MiB, cmd/object-api-common.go:34, moved into a pool that writes blockSizeV2 = 1 MiB blocks).
 * The part is still read, verified and failed over in source blocks; each source block becomes R destination blocks.
 * Refused before any device work: src == dst or a NULL src / dst / files / out_files (MEC_ERR_INVALID_ARGUMENT; for the same
 * geometry use a second handle), a dst block size that does not divide src's (larger ones included), different devices, or an
 * algorithm other than HighwayHash256S on either side (MEC_ERR_UNSUPPORTED: whole-file bitrot chains one digest over the whole
 * shard file, so such parts move through mec_transcode_whole), fewer than write_quorum non-NULL out_files
 * (MEC_ERR_WRITE_QUORUM).  total_length == 0 returns 0 and
 * writes nothing.  Fewer than k readable source files is MEC_ERR_READ_QUORUM.  Both codecs are held for the call.  Counters:
 * "blocks_read" and "bytes_h2d" grow on src, "blocks_encoded" and "bytes_d2h" on dst. */
int64_t mec_transcode(mec_codec* src, const uint8_t* const* files, const uint8_t* prefer, int64_t total_length,
                      mec_codec* dst, uint8_t* const* out_files, int write_quorum, int* heal_hint);

/* ---- cross-request coalescer: many concurrent PutObject calls, one launch ---------------------------------------------------
 * MinIO encodes one block per loop iteration on every request goroutine (cmd/erasure-encode.go:76-108, one Erasure per request,
 * cmd/erasure-object.go:1371); a launch that small leaves 131 of 132 SMs idle.  A batcher owns one codec (k, m, block_size,
 * HighwayHash256S) and a worker thread: callers block in mec_batcher_encode / mec_batcher_encode_sg (same arguments and results
 * as mec_encode / mec_encode_sg), the worker merges everything that is queued — up to max_batch_blocks erasure blocks, waiting
 * at most max_wait_us for company when the GPU is idle — into one staged buffer (one batched copy call) and ONE fused launch over
 * all full blocks, then writes every caller's frames straight into that caller's buffers.  Up to six merged batches are in flight;
 * device staging for all six is allocated here (about 2.4 x max_batch_blocks x block_size each).
 * mec_batcher_stat: "batches", "requests", "blocks", "kernel_batches" (batches moved by the gather / scatter kernels), "redone"
 * (merged GETs and heals that met a frame failing its digest check and were redone on their own), "crc_requests" (PUTs through
 * mec_batcher_encode_crc / _sums with a non-empty CRC mask that got their checksums), "sum_requests" (PUTs through
 * mec_batcher_encode_sums that got at least one MD5 / SHA-1 / SHA-256 digest), "launches", "patterns" (distinct erasure patterns — reader
 * set plus rebuilt shards — summed over GET and heal batches) and "mixed_batches" (GET and heal batches of more than one pattern);
 * with MEC_BATCHER_TRACE=1 in the environment also the worker's and the streams' accumulated phase times "us_submit", "us_sync",
 * "us_finish", "us_idle", "us_stage", "us_kernel", "us_scatter".  Any other name is answered by mec_get_stat on the batcher's own
 * codec, so "form_*", "last_*", "small_launches", "num_sms" and the rest describe the merged launches.
 * The MEC_BATCHER_* environment switches (MEC_BATCHER_TRACE, MEC_BATCHER_MEMCPY, ...) are read once, when the batcher is created. */
typedef struct mec_batcher mec_batcher;
int mec_batcher_new(int k, int m, int64_t block_size, int device, int64_t max_batch_blocks, int max_wait_us, mec_batcher** out);
/* mec_batcher_new with creation flags (mec_batcher_new is flags = 0); unknown bits return MEC_ERR_INVALID_ARGUMENT.
 * MEC_BATCHER_MIX_PATTERNS: GETs merge with GETs and heals with heals whatever drives they read and rebuild.  MinIO rotates every
 * object's shard indices over the drives (hashOrder, cmd/erasure-metadata-utils.go:178, applied by getObjectWithFileInfo and
 * healObject: cmd/erasure-object.go:313, cmd/erasure-healing.go:501,511), so with one drive offline or stale, concurrent reads of
 * different objects rarely share a reader set or a stale set, and without the flag they split into one batch per pattern.  With
 * it a batch of several patterns is ONE launch of the latency kernel, every erasure block with its own decode matrix; such a batch
 * is cut at the blocks one latency launch takes (5 per SM), and a single request larger than that keeps a batch of its own.  A
 * codec whose options rule out the latency kernel ignores the flag. */
#define MEC_BATCHER_MIX_PATTERNS 1
int mec_batcher_new_ex(int k, int m, int64_t block_size, int device, int64_t max_batch_blocks, int max_wait_us, int flags,
                       mec_batcher** out);
void mec_batcher_free(mec_batcher* b);
int64_t mec_batcher_encode(mec_batcher* b, const uint8_t* src, int64_t len, uint8_t* const* files, int write_quorum);
int64_t mec_batcher_encode_sg(mec_batcher* b, const uint8_t* src, int64_t len, uint8_t* const* files, uint8_t* data_digests,
                              int write_quorum);
/* A PutObject through the coalescer together with the object checksums hash.Reader computes over the same bytes
 * (internal/hash/reader.go:267-310).  data_digests == NULL: the outputs of mec_batcher_encode (complete part files); non-NULL: those
 * of mec_batcher_encode_sg.  Returns what that call returns.  `which & 7` is a mask of MEC_CRC* (below); out3 receives CRC32,
 * CRC32C and CRC64NVME as in mec_checksums (0 where not asked for), computed on the bytes the merged batch staged in device memory:
 * two more launches per batch that holds such requests, however many, and one small copy back.  out3 is written only when the call
 * returns >= 0 (len == 0: the checksums of the empty stream, all 0); an empty mask is mec_batcher_encode / _sg and out3 may then be
 * NULL; a non-empty mask with out3 == NULL returns MEC_ERR_INVALID_ARGUMENT before anything is queued.  Requests with and without a
 * mask share batches. */
int64_t mec_batcher_encode_crc(mec_batcher* b, const uint8_t* src, int64_t len, uint8_t* const* files, uint8_t* data_digests,
                               int write_quorum, int which, uint64_t* out3);
/* mec_batcher_encode_crc plus the hashes hash.Reader computes over a PutObject body that cannot be merged from parts: MD5 for the
 * ETag (internal/etag/reader.go), SHA-256 of a signed payload (x-amz-content-sha256) and SHA-1 / SHA-256 of x-amz-checksum-sha1 /
 * -sha256 (internal/hash/reader.go:267-310).  Outputs and return value are those of mec_batcher_encode_crc (data_digests == NULL:
 * complete part files; non-NULL: the scatter-gather outputs).  `which` is any subset of MEC_CRC* and MEC_SUM_* (below); any other
 * bit returns MEC_ERR_INVALID_ARGUMENT.  crc3 receives the CRCs as mec_batcher_encode_crc's out3 does; sums (MEC_SUM_BYTES bytes)
 * receives the asked-for digests at their offsets, the other bytes are left as they were.  A set bit with a NULL destination returns
 * MEC_ERR_INVALID_ARGUMENT before anything is queued.  Outputs are written only when the call returns >= 0; len == 0 gives the
 * digests of the empty message without device work.  Each batch that holds requests with MEC_SUM_* bits adds ONE stream_sums_kernel
 * launch (one thread per request and algorithm, on a second stream of the batch's slot, forked once the batch is staged so the
 * encode does not wait for it) and one small copy back; the batch completes when both are done.  Requests with and without hashes
 * share batches. */
int64_t mec_batcher_encode_sums(mec_batcher* b, const uint8_t* src, int64_t len, uint8_t* const* files, uint8_t* data_digests,
                                int write_quorum, int which, uint64_t* crc3, uint8_t* sums);
/* Erasure.Decode through the coalescer (arguments and results of mec_decode): GETs queued together that see the same drives online
 * share one reader set and are merged into one fused launch (gather kernel, reconstruct, scatter into every caller's dst).  A request
 * that meets a corrupt frame is redone on its own with parallelReader's exact fail-over; pageable buffers take the same private path. */
int64_t mec_batcher_decode(mec_batcher* b, const uint8_t* const* files, int64_t offset, int64_t length, int64_t total_length,
                           uint8_t* dst, int* heal_hint);
/* getObjectWithFileInfo's Erasure.Decode with `prefer` (local drives first, cmd/erasure-object.go:387) through the coalescer:
 * arguments and results of mec_decode_prefer; prefer == NULL is mec_batcher_decode.  With `prefer` the readers are chosen on the
 * caller's thread exactly as mec_decode_prefer chooses them, and GETs that read the same k drives share a launch (any GETs on a
 * batcher created with MEC_BATCHER_MIX_PATTERNS).  A request that meets a corrupt frame is redone on its own through
 * mec_decode_prefer with the same `prefer`. */
int64_t mec_batcher_decode_prefer(mec_batcher* b, const uint8_t* const* files, const uint8_t* prefer, int64_t offset, int64_t length,
                                  int64_t total_length, uint8_t* dst, int* heal_hint);
/* Erasure.Heal (cmd/erasure-decode.go:317) through the coalescer (arguments and results of mec_heal_prefer): heals queued together
 * that read the same k drives (the ones parallelReader picks for `files` and `prefer`) and rebuild the same stale drives (out_files[i]
 * != NULL) are merged into one fused launch (any heals with MEC_BATCHER_MIX_PATTERNS), and one scatter kernel writes every healed frame into every caller's out files.  A
 * request whose chosen readers fail a digest check is redone on its own through mec_heal_prefer (MEC_ERR_FILE_CORRUPT, corrupt[]
 * filled, counted in "redone"); pageable buffers, a drive that is both a reader and stale, and sets of more than 32 drives take that
 * private path directly. */
int mec_batcher_heal(mec_batcher* b, const uint8_t* const* files, const uint8_t* prefer, int64_t total_length,
                     uint8_t* const* out_files, uint8_t* corrupt);
/* A batcher that also moves parts from its own geometry (k, m) to a destination geometry (dst_k, dst_m) of the same block size on
 * the same device.  mec_batcher_new_ex with a second, private destination codec; flags as there.  Geometry errors of either side
 * are those of mec_codec_new; dst_k == k && dst_m == m is allowed (rebalance between equal pools).  The batcher still serves
 * mec_batcher_encode*, mec_batcher_decode* and mec_batcher_heal for (k, m) exactly as a mec_batcher_new_ex batcher does.
 * Extra device memory: the destination codec's six slots are sized up front like the source's, each for B = max_batch_blocks
 * + min(64, max_batch_blocks / 8 + 4) blocks: B x (block_size + dst_m x round_up(S', 16) + (dst_k + dst_m) x 32) bytes plus small
 * tables (S' = ceil(block_size / dst_k)) — about 6 x B x block_size x (1 + dst_m / dst_k) in all: 4.5 GiB for RS(6,2) at 1 MiB
 * blocks and max_batch_blocks = 512. */
int mec_batcher_new_transcode(int k, int m, int dst_k, int dst_m, int64_t block_size, int device, int64_t max_batch_blocks,
                              int max_wait_us, int flags, mec_batcher** out);
/* mec_batcher_new_transcode with a destination block size of its own: moves from (k, m, block_size) to (dst_k, dst_m,
 * dst_block_size), where block_size = R x dst_block_size for an integer R >= 1 (mec_transcode's rule; mec_batcher_new_transcode is
 * dst_block_size = block_size).  Refusals in this order: the source geometry's errors, then the destination's, as mec_codec_new
 * reports them; unknown flags (MEC_ERR_INVALID_ARGUMENT); block_size % dst_block_size != 0 (MEC_ERR_UNSUPPORTED).
 * max_batch_blocks, the private-path threshold and the 1 GiB cap on a merged batch's staging count source blocks.  The destination
 * codec's six slots are sized for the object bytes of a full source batch: B x R destination blocks each (B as above), i.e.
 * B x R x (dst_block_size + dst_m x round_up(S', 16) + (dst_k + dst_m) x 32) bytes plus small tables (S' = ceil(dst_block_size /
 * dst_k)) — per object byte what an R = 1 batcher spends.  Example: RS(12,4) at 10 MiB into RS(6,2) at 1 MiB (R = 10),
 * max_batch_blocks = 16: B = 16 + 6 = 22, so each destination slot holds 220 blocks, 220 MiB of object bytes plus 73 MiB of
 * parity rows, about 1.7 GiB for all six; the source side's six slots (staging, survivor arena, rebuilt rows) take about 3 GiB
 * more. */
int mec_batcher_new_transcode_ex(int k, int m, int64_t block_size, int dst_k, int dst_m, int64_t dst_block_size, int device,
                                 int64_t max_batch_blocks, int max_wait_us, int flags, mec_batcher** out);
/* mec_transcode through the coalescer: arguments, results, heal_hint and refusals of mec_transcode (files / prefer / total_length
 * of the source, out_files / write_quorum of the destination).  Checked on the caller's thread before anything is queued: a NULL
 * batcher, files or out_files, total_length < 0 or a batcher not made by mec_batcher_new_transcode (MEC_ERR_INVALID_ARGUMENT), fewer
 * than write_quorum non-NULL out_files (MEC_ERR_WRITE_QUORUM), total_length == 0 (returns 0, writes nothing), fewer than k readable
 * source files (MEC_ERR_READ_QUORUM).  The readers are chosen there as parallelReader chooses them (`prefer` first, then index
 * order); moves that read the same k drives share one merged batch (any moves with MEC_BATCHER_MIX_PATTERNS, cut at one latency
 * launch as GET and heal batches are): staged and rebuilt as whole-part GETs, re-split on the device, encoded and scattered as
 * merged PUTs of the destination geometry — the object bytes never leave the device.  A move whose readers fail a digest check is
 * redone on its own with mec_transcode on a private pair of handles (every out file rewritten, heal_hint = MEC_ERR_FILE_CORRUPT,
 * counted in "redone"); moves with a chosen reader or an out file that is not page-locked, geometries of more than 32 drives,
 * MEC_BATCHER_MEMCPY in the environment, and parts of more than max_batch_blocks blocks take that private path directly.
 * mec_batcher_stat: "transcodes" (moves completed by merged batches), "transcodes_serial" (moves of the private path, redos
 * included); names prefixed "dst_" are answered by mec_get_stat on the destination codec ("dst_blocks_encoded", "dst_bytes_d2h",
 * "dst_form_small", "dst_launches", ...).  As with mec_transcode, "blocks_read" and "bytes_h2d" grow on the source codec,
 * "blocks_encoded" and "bytes_d2h" on the destination codec. */
int64_t mec_batcher_transcode(mec_batcher* b, const uint8_t* const* files, const uint8_t* prefer, int64_t total_length,
                              uint8_t* const* out_files, int write_quorum, int* heal_hint);
/* mec_transcode_whole through the coalescer, on any batcher made by mec_batcher_new_transcode or mec_batcher_new_transcode_ex: the
 * source geometry (k, m, block_size) is the batcher's, the destination its destination codec (whose block size may divide the
 * source's, as for mec_batcher_transcode).  algo is the part's whole-file algorithm (MEC_SHA256, MEC_BLAKE2B512 or
 * MEC_HIGHWAYHASH256), files[i] the raw shard file of source drive i (NULL = offline), sums + i*64 its expected digest
 * (erasure.GetChecksumInfo(part.Number).Hash); prefer, out_files, write_quorum, heal_hint and the result as mec_transcode_whole.
 * Checked on the caller's thread before anything is queued, in this order: a NULL batcher, files, sums or out_files,
 * total_length < 0, a batcher not made for transcoding, or an algo that is no MEC_* bitrot value (MEC_ERR_INVALID_ARGUMENT,
 * *heal_hint = 0); MEC_HIGHWAYHASH256S (MEC_ERR_UNSUPPORTED: a streaming part moves through mec_batcher_transcode); fewer than
 * write_quorum non-NULL out_files (MEC_ERR_WRITE_QUORUM); total_length == 0 (returns 0, writes nothing); fewer than k non-NULL
 * source files (MEC_ERR_READ_QUORUM).  The k readers are chosen there as parallelReader chooses them (`prefer` first, then index
 * order).  A merged batch holds whole-file moves of one algorithm only, never other kinds of requests; without
 * MEC_BATCHER_MIX_PATTERNS its moves share one reader set, with it reader sets mix and the batch is cut at one latency launch.
 * A batch stages the chosen readers' shard files of all its moves in one batched copy, hashes all of them in ONE whole_hash_kernel
 * launch (one thread per file, two for HighwayHash256: a batch waits for its longest file), rebuilds the missing data shards from
 * the raw rows in one merged reconstruct, and re-splits, encodes and scatters as mec_batcher_transcode does.  A move whose chosen
 * readers all match their sums is done (heal_hint = 0, counted in "transcodes_whole").  A move with any mismatching reader is
 * redone alone on the private pair, which applies the exact fail-over (the next reader in `prefer` order, heal_hint =
 * MEC_ERR_FILE_CORRUPT, every out file rewritten; counted in "redone" and "transcodes_whole_serial").  Moves with a chosen reader
 * or an out file that is not page-locked, geometries of more than 32 drives, MEC_BATCHER_MEMCPY in the environment and parts of
 * more than max_batch_blocks source blocks take that private path directly: mec_transcode_whole on a private source handle of the
 * request's algorithm (up to three, each created on first use) and the private destination handle.  As for mec_batcher_transcode,
 * the out files' contents are unspecified when the call returns an error.
 * Counters (mec_batcher_stat): "transcodes_whole" (moves completed by merged batches), "transcodes_whole_serial" (moves of the
 * private path, redos included); "whole_hash_launches" grows by one per merged whole-file batch; "blocks_read" and "bytes_h2d"
 * (k x mec_shard_file_size(total_length) per clean move) grow on the source side, "dst_blocks_encoded" and "dst_bytes_d2h" on the
 * destination side.  Device memory: the file arena of a batch (its object bytes plus at most 272 x k bytes per request) is the
 * source slot's PUT staging buffer, which mec_batcher_new_transcode* sizes up front for a full batch: max_batch_blocks +
 * min(64, max_batch_blocks / 8 + 4) blocks of block_size + 272 x k bytes (at 1 MiB blocks within the slack the PUT staging
 * already has), plus a 16-byte stream-table entry and a 64-byte digest per staged file. */
int64_t mec_batcher_transcode_whole(mec_batcher* b, int algo, const uint8_t* const* files, const uint8_t* sums,
                                    const uint8_t* prefer, int64_t total_length, uint8_t* const* out_files, int write_quorum,
                                    int* heal_hint);
/* mec_decode_mixed / mec_heal_mixed through the coalescer, on any batcher (its codec is the HighwayHash256S codec of the part's
 * geometry): the arguments of those calls with the batcher in place of the codec, and their results, heal_hint and corrupt[].
 * Checked on the caller's thread before anything is queued, in the single-codec calls' order: a NULL batcher, algos or files (heal:
 * out_files) (MEC_ERR_INVALID_ARGUMENT, *heal_hint = 0); for decode the range checks, length == 0 (returns 0), a NULL dst and
 * MEC_ERR_SHORT_DATA; the drive formats (an algos[i] that is no MEC_* value, or a NULL sums beside a whole-file read drive:
 * MEC_ERR_INVALID_ARGUMENT; two whole-file algorithms: MEC_ERR_UNSUPPORTED); heal with total_length <= 0 (MEC_OK); fewer than k
 * readable drives (MEC_ERR_READ_QUORUM).  The k readers are chosen there as mec_decode_mixed chooses them: drives with files[i] !=
 * NULL (heal: and out_files[i] == NULL), `prefer` first, then index order.
 * A call whose k chosen readers all stream is an ordinary merged GET or heal: it shares batches with mec_batcher_decode_prefer /
 * mec_batcher_heal requests under their rules.  A call with a whole-file reader among them joins batches of such calls of the same
 * whole-file algorithm only (without MEC_BATCHER_MIX_PATTERNS of the same reader set — and, for heals, stale set — with it of any,
 * cut at one latency launch).  Such a batch stages the streaming readers' frames of every range as GET batches do and the
 * whole-file readers' entire shard files into a file arena, hashes all those files in ONE whole_hash_kernel launch, lays their raw
 * rows into the frame arena and runs the merged reconstruct and scatters unchanged (a GET batch in which no call reads frames skips
 * the frame digests, and launches nothing more when nothing is rebuilt).  A call whose streaming frames pass their digests and whose
 * whole-file readers match their sums is done (counted in "reads_whole" when it has a whole-file reader); any other is redone alone
 * through mec_decode_mixed / mec_heal_mixed with the same `prefer` on the batcher's private handle, which applies parallelReader's
 * exact fail-over (counted in "redone" and "reads_whole_serial"), and its batch neighbours complete as merged.  Calls with a chosen
 * reader, dst or out file that is not page-locked, more than 32 drives, MEC_BATCHER_MEMCPY in the environment, more stale drives
 * than a merged heal rebuilds, or a whole-file reader and a part of more than max_batch_blocks blocks take that private path
 * directly (counted in "reads_whole_serial").
 * Counters: "whole_hash_launches" grows by one per merged batch with whole-file readers; such a batch adds to "bytes_h2d" what
 * mec_decode_mixed would (the frame bytes of every streaming reader plus one shard file per whole-file reader), and to
 * "blocks_read" and "shards_rebuilt" what every merged read batch adds.
 * Device memory: a slot's first batch with whole-file readers sizes its file arena for a full batch — B x (block_size + 272 x k)
 * bytes in the PUT staging buffer (B = max_batch_blocks + min(64, max_batch_blocks / 8 + 4)), plus 84 bytes of stream table,
 * digest and pinned mirrors per file slot, B x k of them — and later batches allocate nothing.  Transcode batchers have it from
 * the start; a batcher that never sees a whole-file reader allocates nothing more.  GET batches with whole-file readers scatter
 * straight into the callers' buffers, since the file arena takes the staging buffer the GET assembly would use. */
int64_t mec_batcher_decode_mixed(mec_batcher* b, const int* algos, const uint8_t* const* files, const uint8_t* sums,
                                 const uint8_t* prefer, int64_t offset, int64_t length, int64_t total_length, uint8_t* dst,
                                 int* heal_hint);
int mec_batcher_heal_mixed(mec_batcher* b, const int* algos, const uint8_t* const* files, const uint8_t* sums,
                           const uint8_t* prefer, int64_t total_length, uint8_t* const* out_files, uint8_t* corrupt);
/* mec_bitrot_verify_parts through the coalescer (VerifyFile of one object on one drive, cmd/xl-storage.go:3100-3137; the deep-scan
 * heals of the scanner, MRF and HealObject send many of them at once, cmd/erasure-healing-common.go:415-419), on any batcher
 * (transcode batchers included): the arguments and results of mec_bitrot_verify_parts with the batcher in place of the codec; streaming
 * parts use the batcher's shard size.  Checked on the caller's thread, before anything is queued and in this order: a NULL batcher,
 * then mec_bitrot_verify_parts' refusals (MEC_ERR_INVALID_ARGUMENT, results untouched), then its per-part decisions (invalid parts,
 * wrong streaming lengths, empty streaming parts); a call with nothing left to hash returns MEC_OK at once.
 * Calls with a file to hash that is not page-locked, MEC_BATCHER_MEMCPY in the environment, more frames than one hash-only launch of
 * the latency kernel takes (its "small_blocks" limit; B when the codec's options rule that kernel out), more staged bytes than
 * B x block_size - 1024 (a frame pitch of round_up(32 + S, 16) per frame, round_up(file_len, 16) + 256 per whole-file part) or more
 * whole-file parts than B x k (B = max_batch_blocks + min(64, max_batch_blocks / 8 + 4)) run through mec_bitrot_verify_parts on the
 * batcher's private handle (counted in "verifies_serial").  Every other call joins a merged verify batch: verify calls only, and calls
 * with a whole-file part only with such calls, whatever their algorithms (a frame-only scan never waits behind the chain hash of a
 * long legacy file); a batch is cut at those same frame, byte and file limits.  A batch stages every frame and every whole file in
 * ONE batched copy, hashes every frame in ONE hash-only launch with a per-frame length table (one launch per run of full frames and
 * one per short frame when the options rule out the latency kernel) and every whole file in ONE whole_hash_kernel launch of up to
 * three algorithm groups, and copies the verdicts and digests back once.  Nothing is redone: a corrupt part is a result and never
 * affects its batch neighbours.
 * Counters (mec_batcher_stat): "verifies" (calls completed by merged batches), "verifies_serial"; "batches", "requests" and "launches"
 * as for other kinds; "blocks_read" grows by the frames hashed, "bytes_h2d" by the bytes staged (file_lens of every hashed part),
 * "whole_hash_launches" by one per batch with whole-file parts.  Device memory: frames and files are staged in the slot's PUT
 * staging buffer, which mec_batcher_new* sizes; a slot's first batch with whole-file parts sizes its file arena and stream table as
 * mec_batcher_decode_mixed does (size shared with those batches), and the per-frame length table and verdict buffers grow to the
 * largest batch; nothing more is allocated when the batcher is created. */
int mec_batcher_verify(mec_batcher* b, int64_t nparts, const int* algos, const uint8_t* const* files, const int64_t* file_lens,
                       const int64_t* part_lens, const uint8_t* sums, int* results);
/* mec_encode_sse / mec_decode_sse (below) through the coalescer: arguments, results, part files and refusals are theirs, with the
 * batcher in place of the codec, and every refusal is made on the caller's thread before anything is queued.
 * mec_batcher_encode_sse joins merged PUT batches (encrypted and plain PUTs share them) as its ciphertext of
 * mec_dare_encrypted_size(len) bytes, which max_batch_blocks and the wake rule count.  A batch stages the plain requests and the
 * encrypted requests' plaintext in ONE batched copy (the plaintext into a per-slot arena), runs ONE key-setup launch and ONE seal
 * launch over every package of every encrypted request (each package sealed once, into a per-request ciphertext arena), moves each
 * ciphertext into its place in the batch layout in one batched device-to-device copy, and encodes and scatters as for plain PUTs.
 * Returns len.
 * mec_batcher_decode_sse maps [offset, offset + length) to the ciphertext range of its whole packages and reads that range as an
 * ordinary merged GET of the part (reader sets as mec_batcher_decode_prefer; any with MEC_BATCHER_MIX_PATTERNS); the batch assembles
 * every encrypted request's ciphertext on the device, runs ONE key-setup and ONE open launch over every package, and copies each
 * request's plaintext range back in one batched copy.  A request that met a frame failing its digest is redone alone through
 * mec_decode_sse on the private handle (counted in "redone"); otherwise a package the request may not open (DARE 1.0; ChaCha20-
 * Poly1305 at option "dare_chacha20" 0) returns MEC_ERR_UNSUPPORTED and any other failing package MEC_ERR_NOT_AUTHENTIC, with
 * dst[0, length) zeroed.  One request's failure never affects its batch neighbours.
 * Option "dare_chacha20" (mec_batcher_set_option): each encrypted request records the batcher's value when it is admitted and runs
 * under it, in whichever batch it merges and when it is redone alone; one batch may hold requests admitted under different values.
 * A GET batch with a request at 1 or 2 adds ONE ChaCha20-Poly1305 open launch behind the AES one, which opens the cipher-1 packages
 * of exactly those requests.  A PUT batch seals the packages of its requests at 2 with ONE ChaCha20-Poly1305 launch, and those of the
 * others with the AES one; a batch whose encrypted requests are all at 2 has no setup and no AES launch.
 * Calls whose buffers are not page-locked, and MEC_BATCHER_MEMCPY, run through mec_encode_sse / mec_decode_sse on the private handle.
 * Each slot holds its own key table: the device copy is zeroed on the slot's stream behind the batch's cipher launch, the host copy
 * before any caller of the batch is woken, and no pointer to a caller's key outlives the call.  Device memory: each slot's plaintext
 * arena is sized on its first encrypted batch for a full batch, B x block_size bytes (B = max_batch_blocks + min(64,
 * max_batch_blocks / 8 + 4); with six slots, 6 x B x block_size in all), and grows past that only for a batch led by a request of
 * more than B blocks; a PUT batch's ciphertext arena is the slot's survivor arena, which mec_batcher_new* sizes and PUT batches do
 * not otherwise use.  The codec's AES tables are built, to completion, by the first encrypted batch.
 * Counters (mec_batcher_stat): "sse_puts" and "sse_gets" (calls completed by merged batches), "sse_serial" (calls of the private
 * path, redos included); "dare_sealed", "dare_opened", "dare_chacha20" and "launches" are the batcher codec's. */
int64_t mec_batcher_encode_sse(mec_batcher* b, const uint8_t* src, int64_t len, const uint8_t key[32], const uint8_t nonce[12],
                               uint8_t* const* files, int write_quorum);
int64_t mec_batcher_decode_sse(mec_batcher* b, const uint8_t* const* files, const uint8_t* prefer, int64_t offset, int64_t length,
                               int64_t enc_total, const uint8_t key[32], uint8_t* dst, int* heal_hint);
int64_t mec_batcher_stat(const mec_batcher* b, const char* name);
/* Options of a batcher: only "dare_chacha20" (0, 1 or 2, as mec_set_option), applied to the batcher's codec and its private handle;
 * requests admitted afterwards run under the new value.  A NULL batcher or name, another name or another value is
 * MEC_ERR_INVALID_ARGUMENT and changes nothing. */
int mec_batcher_set_option(mec_batcher* b, const char* name, int64_t value);

/* ---- object checksums of the PutObject stream (internal/hash/checksum.go:64-73, internal/hash/crc.go) ---------------------
 * CRC32 (IEEE), CRC32C (Castagnoli) and CRC64NVME — the checksum types hash.Reader can merge (ChecksumType.CanMerge) — of a
 * byte stream, as the finalized values Go's hash/crc32 and hash/crc64 return (big-endian encode them for Checksum.Raw).
 * `which` is a mask of MEC_CRC*; out3[0] = CRC32, out3[1] = CRC32C, out3[2] = CRC64NVME (0 where not asked for).
 *   mec_checksums_device : the stream is already in device memory (e.g. staged for an encode)
 *   mec_checksums        : host buffer, staged through the codec's slots
 *   mec_checksum_combine : Checksum.AddPart (crc.go:32-73): checksum of A || B from those of A and B and |B|, on the host
 * mec_set_option(c, "checksums", mask) makes mec_encode / mec_encode_sg / mec_encode_blocks compute them on the bytes they stage
 * anyway (the object crosses PCIe once); mec_last_checksums returns the values of the codec's last such call and its length
 * (an empty object included: (0, 0, 0) and 0). */
#define MEC_CRC32 1
#define MEC_CRC32C 2
#define MEC_CRC64NVME 4
int mec_checksums_device(mec_codec* c, const uint8_t* d_src, int64_t len, int which, uint64_t* out3, void* cuda_stream);
int mec_checksums(mec_codec* c, const uint8_t* src, int64_t len, int which, uint64_t* out3);
uint64_t mec_checksum_combine(int type, uint64_t crc1, uint64_t crc2, int64_t len2);
int64_t mec_last_checksums(const mec_codec* c, uint64_t* out3);

/* ---- object hashes of many messages at once (MD5, SHA-1, SHA-256) ----------------------------------------------------------
 * MD5 (the ETag), SHA-1 and SHA-256 are chains that cannot be split: one GPU thread hashes one message, far slower than a CPU core
 * does, so this pays only for many independent messages at once (one thread per message and algorithm, one launch).
 * mec_sums_device: message i is d_base[offsets[i], offsets[i] + lens[i]) (offsets and lens are host arrays, read before the call
 * returns; any byte alignment); its record is d_sums + i * MEC_SUM_BYTES: MD5 at +0 (16 bytes), SHA-1 at +32 (20 bytes), SHA-256 at
 * +64 (32 bytes), each in the byte order of Go's Sum(nil).  Slots of algorithms not asked for, and the padding bytes, are left as
 * they were.  `which` must be a non-empty subset of MEC_SUM_*; any other value, count < 0, a negative offset or length, or NULL
 * offsets / lens / d_sums with count > 0 (or d_base with a non-empty message) return MEC_ERR_INVALID_ARGUMENT before any device
 * work.  A zero-length message yields the digest of the empty message.  Asynchronous on `cuda_stream`; calls on one handle share
 * its work table, so a call first waits on the host until the previous call's kernel has finished. */
#define MEC_SUM_MD5 8
#define MEC_SUM_SHA1 16
#define MEC_SUM_SHA256 32
#define MEC_SUM_BYTES 96 /* MD5 at +0 (16 B), SHA-1 at +32 (20 B), SHA-256 at +64 (32 B) */
int mec_sums_device(mec_codec* c, int which, const uint8_t* d_base, const int64_t* offsets, const int64_t* lens, int64_t count,
                    uint8_t* d_sums, void* cuda_stream);

/* ---- legacy whole-file bitrot (cmd/bitrot-whole.go, BitrotAlgorithm SHA256 / BLAKE2b512 / HighwayHash256) ----
 * Erasure.Encode with wholeBitrotWriters (cmd/bitrot-whole.go:35-45): files[i] receives the raw shard file
 * (shards of all blocks back to back, mec_shard_file_size(len) bytes) and sums + i*64 the digest over the whole
 * file that bitrotWriterSum (cmd/bitrot.go:148) would return (32 or 64 bytes).  The codec's algorithm must be
 * one of the whole-file algorithms.  Returns bytes consumed. */
int64_t mec_encode_whole(mec_codec* c, const uint8_t* src, int64_t len, uint8_t* const* files, uint8_t* sums,
                         int write_quorum);
/* BitrotAlgorithm.New() hash.Hash one-shot (cmd/bitrot.go:47-64) for a whole-file algorithm: digests of
 * `count` equal-length messages laid out back to back; digest i at digests + i*mec_digest_size(algo).
 * Also bitrotVerify's non-streaming branch (cmd/bitrot.go:165-175): hash the file, compare with `want`. */
int mec_whole_hash(mec_codec* c, int algo, const uint8_t* msgs, int64_t msg_len, int64_t count, uint8_t* digests);
int mec_bitrot_verify_whole(mec_codec* c, int algo, const uint8_t* file, int64_t file_len, const uint8_t* want);
/* Device-resident mec_whole_hash: message i at d_msgs + i*pitch (pitch a multiple of 16, >= msg_len, with 128 readable
 * bytes after the last message), digest i at d_digests + i*64 (bytes digest_size..63 of each slot are left as they were).
 * d_msgs must be 16-byte aligned (NULL only when msg_len or count is 0) and d_digests non-NULL and 8-byte aligned; other
 * pointers return MEC_ERR_INVALID_ARGUMENT before any device work.  Asynchronous on `cuda_stream`. */
int mec_whole_hash_device(mec_codec* c, int algo, const uint8_t* d_msgs, int64_t pitch, int64_t msg_len, int64_t count,
                          uint8_t* d_digests, void* cuda_stream);
/* Erasure.Decode / Erasure.Heal over whole-file bitrot readers (wholeBitrotReader.ReadAt, cmd/bitrot-whole.go:66-81): files[i] is
 * the RAW shard file of drive i (mec_shard_file_size(total) bytes, NULL = offline), sums + i*64 its expected digest (the
 * checksum xl.meta keeps for whole-file algorithms).  A reader whose whole-file digest does not match is errFileCorrupt: it is
 * dropped and the next drive in index order takes its place (cmd/xl-storage.go:1931-1950, cmd/erasure-decode.go:196-199).
 * mec_decode_whole returns bytes written (*heal_hint = MEC_ERR_FILE_CORRUPT when a reader was dropped but the read succeeded).
 * mec_heal_whole rebuilds every shard file with out_files[i] != NULL, writes its digest to out_sums + i*64 (optional) and returns
 * MEC_OK, or MEC_ERR_FILE_CORRUPT when it healed but met bitrot in a source (corrupt[i], optional, names the readers).
 * The codec's algorithm must be SHA256, BLAKE2b512 or HighwayHash256.  mec_heal_whole writes the legacy format (raw shard files
 * and whole-file sums); healObject heals into the streaming format, which is what mec_heal_mixed writes. */
int64_t mec_decode_whole(mec_codec* c, const uint8_t* const* files, const uint8_t* sums, int64_t offset, int64_t length,
                         int64_t total_length, uint8_t* dst, int* heal_hint);
int mec_heal_whole(mec_codec* c, const uint8_t* const* files, const uint8_t* sums, int64_t total_length,
                   uint8_t* const* out_files, uint8_t* out_sums, uint8_t* corrupt);
int mec_digest_size(int algo);

/* mec_transcode for a part written with a whole-file bitrot algorithm (the oldest parts, mostly with blockSizeV1 = 10 MiB blocks,
 * which decommission and rebalance drain): the source side has mec_decode_whole's meaning over the whole part — files[i] the raw
 * shard file of drive i (NULL = offline), sums + i*64 its expected digest (erasure.GetChecksumInfo(part.Number).Hash) — with
 * mec_decode_prefer's `prefer` (readers with prefer[i] != 0 first, as parallelReader.preferReaders orders them).  A reader whose
 * whole-file digest does not match is dropped and the next one in that order takes its place; the call then still moves the part
 * and sets *heal_hint = MEC_ERR_FILE_CORRUPT.  out_files / write_quorum as mec_transcode: complete streaming-bitrot part.N images of
 * dst's geometry.  Returns total_length, or a negative MEC_ERR_*.
 * Refused before any device work: src == dst or a NULL src / dst / files / sums / out_files, total_length < 0
 * (MEC_ERR_INVALID_ARGUMENT); a src algorithm other than SHA256, BLAKE2b512 or HighwayHash256 (a streaming part moves through
 * mec_transcode), a dst algorithm other than HighwayHash256S, a dst block size that does not divide src's, or different devices
 * (MEC_ERR_UNSUPPORTED); fewer than write_quorum non-NULL out_files (MEC_ERR_WRITE_QUORUM).  total_length == 0 returns 0 and writes
 * nothing.  The chosen readers are staged and verified before anything is written: fewer than k verified readers is
 * MEC_ERR_READ_QUORUM with every out file untouched.  The readers of a round are hashed by ONE whole_hash_kernel launch (one thread
 * per file: on a move with no corrupt reader the only hash launch of the call), the missing data shards are rebuilt from the raw
 * shard rows, and the part is re-split, encoded and written in chunks of about 32 MiB of object bytes through both codecs' slots.
 * Device memory: the staged source, k x (round_up(mec_shard_file_size(total_length), 16) + 256) bytes in src's slot 0 (as
 * mec_decode_whole), the rebuilt data-shard rows of the chunks in flight on src, and dst's chunk buffers (object bytes, parity rows
 * and digests of a chunk per slot).  Counters: "blocks_read", "bytes_h2d" (k x the shard file size when no reader is dropped) and
 * "corrupt_shards" grow on src, "blocks_encoded" and "bytes_d2h" on dst; src's "bytes_d2h" does not grow. */
int64_t mec_transcode_whole(mec_codec* src, const uint8_t* const* files, const uint8_t* sums, const uint8_t* prefer,
                            int64_t total_length, mec_codec* dst, uint8_t* const* out_files, int write_quorum, int* heal_hint);

/* Erasure.Decode / Erasure.Heal over a part whose drives mix bitrot formats: a legacy part (whole-file algorithm) of which some
 * drives were healed.  healObject heals into HighwayHash256S frames (cmd/erasure-healing.go:593-596) and leaves the healed drive no
 * checksum entry, so it reads as streaming (cmd/erasure-metadata.go:43-51); every GET opens each drive with its own algorithm
 * (cmd/erasure-object.go:381-384) and parallelReader mixes the two reader kinds in one decode.
 *   c          : a HighwayHash256S codec of the part's geometry (another algorithm: MEC_ERR_UNSUPPORTED)
 *   algos[i]   : drive i's bitrot algorithm, read only where files[i] != NULL (heal: and out_files[i] == NULL)
 *                MEC_HIGHWAYHASH256S: files[i] is the drive's part.N image from its first frame, as mec_decode_prefer takes it;
 *                MEC_SHA256, MEC_BLAKE2B512, MEC_HIGHWAYHASH256: files[i] is the raw shard file (mec_shard_file_size(total) bytes),
 *                sums + i*64 its expected digest
 *   prefer     : as mec_decode_prefer; NULL = index order
 * Fail-over is parallelReader's over both kinds.  Readers are chosen as mec_decode_prefer chooses them, preferred ones first, then
 * index order.  A whole-file reader is verified when it is first chosen, before any block is read through it (xlStorage.ReadFile
 * hashes the whole file on the first ReadAt, cmd/xl-storage.go:1931-1950): the whole-file readers that join the set in one round
 * are staged and hashed by ONE whole_hash_kernel launch, and one whose digest does not match is dropped for the rest of the call,
 * corrupt[i] set, and the next reader chosen.  A streaming reader is checked frame by frame; when one fails at block b it is
 * dropped and the call resumes at b with the next reader, which, if it is whole-file, is hashed first.  Whole-file readers that are
 * never chosen are never staged, hashed or reported.  Verified files stay on the device for the whole call:
 * k x (round_up(mec_shard_file_size(total_length), 16) + 256) bytes in a buffer of the codec's own.
 * mec_decode_mixed has mec_decode_prefer's argument checks, in its order (MEC_ERR_SHORT_DATA included), and its results:
 * *heal_hint = MEC_ERR_FILE_CORRUPT when a reader was dropped.
 * mec_heal_mixed: out_files[i] != NULL marks a stale drive, which is never read whatever files[i] holds (healObject opens no reader
 * on a drive it heals, cmd/erasure-healing.go:572-575); it receives the complete HighwayHash256S part.N image, byte for byte what
 * mec_encode writes for drive i.  Returns MEC_OK, MEC_ERR_FILE_CORRUPT (healed, but a reader was dropped; corrupt[i], optional,
 * names them) or MEC_ERR_READ_QUORUM; out files are complete only on the first two.  No whole-file sums come back: a healed drive
 * has none.
 * Refused before any device work: a NULL c, algos or files, for heal a NULL out_files, an algos[i] that is no MEC_* bitrot value on a
 * read drive, a NULL sums while a read drive is whole-file (MEC_ERR_INVALID_ARGUMENT); two different whole-file algorithms among the
 * read drives (MEC_ERR_UNSUPPORTED).  length == 0 returns 0; heal with total_length <= 0 returns MEC_OK.
 * With every drive HighwayHash256S (and no stale drive among the readers) the calls equal mec_decode_prefer / mec_heal_prefer; with
 * every drive whole-file and prefer == NULL, mec_decode_mixed equals mec_decode_whole.
 * Counters: "blocks_read", "shards_rebuilt", "corrupt_shards" and "bytes_d2h" as the streaming calls; "bytes_h2d" = frame bytes of
 * streaming readers + one shard file per whole-file reader hashed; "whole_hash_launches" + 1 per round with whole-file newcomers. */
int64_t mec_decode_mixed(mec_codec* c, const int* algos, const uint8_t* const* files, const uint8_t* sums, const uint8_t* prefer,
                         int64_t offset, int64_t length, int64_t total_length, uint8_t* dst, int* heal_hint);
int mec_heal_mixed(mec_codec* c, const int* algos, const uint8_t* const* files, const uint8_t* sums, const uint8_t* prefer,
                   int64_t total_length, uint8_t* const* out_files, uint8_t* corrupt);

/* bitrotVerify (cmd/bitrot.go:164) for the streaming algorithm: scans a whole shard file. */
int mec_bitrot_verify(mec_codec* c, const uint8_t* file, int64_t file_len, int64_t part_len);
/* The same for many shard files at once (the deep scan of the data scanner visits every part on every drive): results[f] = MEC_OK or
 * MEC_ERR_FILE_CORRUPT (wrong length or a frame that fails its digest); the frames of all files stream through the codec's slots and
 * consecutive full frames — across files — share one hash-only launch.  Returns MEC_OK unless the call itself failed. */
int mec_bitrot_verify_batch(mec_codec* c, int64_t nfiles, const uint8_t* const* files, const int64_t* file_lens,
                            const int64_t* part_lens, int* results);
/* VerifyFile (cmd/xl-storage.go:3100-3137) in one call: bitrotVerify (cmd/bitrot.go:164-216) of every part of an object on one drive,
 * each part with its own algorithm and sum (erasure.GetChecksumInfo(part.Number)), or of xl.meta inline data
 * (cmd/erasure-healing-common.go:398-406).  Part p: algos[p] = checksumInfo.Algorithm, files[p] = file_lens[p] bytes of part.N as
 * stored (or of the inline data), part_lens[p] = erasure.ShardFileSize(part.Size), sums + p*64 = checksumInfo.Hash (read only for
 * whole-file algorithms).  The codec's own algorithm is not used.
 *   streaming (MEC_HIGHWAYHASH256S): frames of the codec's shard size; results[p] is bitrotVerify's verdict: a file length other than
 *     mec_bitrot_shard_file_size(part_lens[p]) or any frame failing its digest is MEC_ERR_FILE_CORRUPT (cmd/bitrot.go:183); an empty
 *     part with an empty file is MEC_OK.
 *   whole-file (MEC_SHA256, MEC_HIGHWAYHASH256, MEC_BLAKE2B512): the digest of all file_lens[p] bytes is compared with the first
 *     mec_digest_size(algo) bytes of the sum (cmd/bitrot.go:165-174); part_lens[p] is not read.
 * Refused before any device work with MEC_ERR_INVALID_ARGUMENT and results untouched, in this order: a NULL codec; nparts < 0; a NULL
 * algos, files, file_lens, part_lens or results while nparts > 0; a NULL sums while a part is whole-file.  Per part, results[p] =
 * MEC_ERR_INVALID_ARGUMENT for an algos[p] that is no MEC_* bitrot value, a negative file_lens[p] (or part_lens[p] of a streaming
 * part), or a NULL files[p] with file_lens[p] > 0.  Returns MEC_OK unless the call itself failed.
 * Streaming parts run through mec_bitrot_verify_batch's pipeline (hash-only launches over ~32 MiB chunks of frames through the codec's
 * slots).  Whole-file parts are staged in input order in groups of at most 256 MiB of file bytes (a larger file alone), each group by
 * ONE batched copy into slot 0's staging buffer (each file 16-byte aligned with 256 bytes behind it) and ONE whole_hash_kernel launch
 * whose up to three algorithm groups hold its SHA256, HighwayHash256 and BLAKE2b512 parts ("whole_hash_launches" + 1 per group).
 * Counters: "blocks_read" grows by the frames hashed, "bytes_h2d" by the file bytes staged.  mec_bitrot_verify_batch is this call
 * with every part MEC_HIGHWAYHASH256S on a HighwayHash256S codec, except that it refuses a NULL file with part_lens[f] > 0 per file. */
int mec_bitrot_verify_parts(mec_codec* c, int64_t nparts, const int* algos, const uint8_t* const* files, const int64_t* file_lens,
                            const int64_t* part_lens, const uint8_t* sums, int* results);

/* ---- server-side encryption: DARE 2.0 packages (minio/sio v0.4.1, AES-256-GCM and ChaCha20-Poly1305) ---------------------------
 * sio.EncryptReader with Version20 (newEncryptReader, cmd/encryption-v1.go:417-428) and DecryptBlocksRequestR (:572).  A package is
 * header[16] = 0x20 | cipher | uint16 LE (payload_len - 1) | nonce[12], the ciphertext and a 16-byte tag; every package but the last
 * carries 65536 bytes, bit 7 of header[4] marks the final one, the AEAD nonce is header[4:16] with bytes 8..11 (uint32 LE) XORed with
 * the sequence number, the additional data header[0:4].  Keys come from the caller (KMS, sealing and DerivePartKey stay in Go) and
 * only the raw key goes to the device, whose setup launch expands it; the key schedule and H powers of a call are zeroed on the device and the host before it returns.
 * Option "dare_chacha20" (mec_set_option) picks the AEAD of header[1]:
 *   0 (default) seals AES-256-GCM (cipher 0); a ChaCha20-Poly1305 package (cipher 1) is MEC_ERR_UNSUPPORTED and gets no plaintext.
 *   1 seals AES-256-GCM and opens every package with the AEAD its own header names (0 or 1; RFC 8439 §2.8 for cipher 1, with the
 *     same nonce and additional data).  An open runs ONE more launch, behind the AES one over the same rows.
 *   2 as 1, and every seal (mec_dare_device, mec_encode_sse, mec_encode_chunked_sse) writes ChaCha20-Poly1305 packages (cipher 1)
 *     with no key-setup launch.
 * At 1 and 2, MEC_ERR_UNSUPPORTED means a DARE 1.0 stream (version 0x10) only; other cipher bytes are MEC_ERR_NOT_AUTHENTIC.
 * Counters: "dare_sealed", "dare_opened" (package rows, each counted once whichever kernels ran it), "dare_chacha20" (the option). */
/* sio.EncryptedSize / DecryptedSize; a negative size, more than 2^32 packages or a remainder of 1..32 bytes is
 * MEC_ERR_INVALID_ARGUMENT. */
int64_t mec_dare_encrypted_size(int64_t n);
int64_t mec_dare_decrypted_size(int64_t enc);
/* Seal or open many streams in device memory in ONE launch (shaped like mec_sums_device).  Stream s: key keys + 32s, first package
 * at sequence number seq0[s].  SEAL: plaintext d_in[in_off[s], + lens[s]) -> packages at d_out + out_off[s], nonce nonces + 12s, the
 * last package final.  OPEN: packages d_in[in_off[s], + lens[s]) -> plaintext at d_out + out_off[s]; enc_totals[s] is the stored size
 * of the part, which fixes each package's length and which one is final.  Each package is checked for version, length, final bit,
 * nonce (the first package's, final bit masked) and tag, and only one that passes gets plaintext written.  status[s] (host): 0, 13
 * (-MEC_ERR_NOT_AUTHENTIC: a package failed, the stored size is no DARE size, or bytes are cut short or run past the part) or 102
 * (-MEC_ERR_UNSUPPORTED: a package of a cipher or version the option does not open).  Returns MEC_ERR_UNSUPPORTED if any stream
 * is, else MEC_ERR_NOT_AUTHENTIC if any failed, else MEC_OK; waits
 * for its work on cuda_stream.  NULL arrays, negative offsets or lengths, an unknown op or a seal past sequence number 2^32 - 1 are
 * MEC_ERR_INVALID_ARGUMENT before any device work. */
#define MEC_DARE_SEAL 1
#define MEC_DARE_OPEN 2
int mec_dare_device(mec_codec* c, int op, int64_t nstreams, const uint8_t* keys, const uint8_t* nonces, const uint32_t* seq0,
                    const int64_t* enc_totals, const uint8_t* d_in, const int64_t* in_off, const int64_t* lens, uint8_t* d_out,
                    const int64_t* out_off, uint8_t* status, void* cuda_stream);
/* EncryptRequest + Erasure.Encode (cmd/object-handlers.go:2070): seals `len` bytes with `key` and the caller's 12 random nonce bytes
 * and writes mec_encode's part files of the sealed stream (sized for mec_dare_encrypted_size(len)).  Returns the plaintext bytes
 * consumed.  "checksums" covers the plaintext.  At option "dare_chacha20" 2 the packages are ChaCha20-Poly1305. */
int64_t mec_encode_sse(mec_codec* c, const uint8_t* src, int64_t len, const uint8_t key[32], const uint8_t nonce[12],
                       uint8_t* const* files, int write_quorum);
/* Erasure.Decode + DecryptBlocksRequestR of one part (multipart callers pass the part key, one call per part): plaintext
 * [offset, offset + length) of a part stored as enc_total bytes; files / prefer / heal_hint as mec_decode_prefer.  Returns length,
 * MEC_ERR_NOT_AUTHENTIC or MEC_ERR_UNSUPPORTED (dst[0, length) zeroed; ChaCha20-Poly1305 packages are UNSUPPORTED at option
 * "dare_chacha20" 0 only, DARE 1.0 always), or mec_decode_prefer's errors.  Each package is opened once; the ciphertext range and its
 * plaintext are held in device buffers of the codec. */
int64_t mec_decode_sse(mec_codec* c, const uint8_t* const* files, const uint8_t* prefer, int64_t offset, int64_t length,
                       int64_t enc_total, const uint8_t key[32], uint8_t* dst, int* heal_hint);

/* ---- Signature V4 streaming payloads (x-amz-content-sha256: STREAMING-AWS4-HMAC-SHA256-PAYLOAD[-TRAILER]) ------------------
 * Each aws-chunk's signature is HMAC-SHA256(signing key, string to sign) over SHA-256 of its payload and the previous chunk's
 * signature (getChunkSignature / getTrailerChunkSignature, cmd/streaming-signature-v4.go:54-94).  `key` is getSigningKey's 32 bytes
 * (cmd/signature-v4.go:141), `date` the request time as "20060102T150405Z" and `scope` "yyyymmdd/region/s3/aws4_request" (NUL-
 * terminated; strlen(date) + strlen(scope) <= 254).  Both calls derive the HMAC chaining states of the key on the host and zero
 * them, device and host copies, before they return.  Counters (mec_get_stat): "sigv4_chunks", rows verified; "sigv4_key_bytes",
 * the non-zero bytes of key material left in the codec (its host copy and a read-back of its device copy), 0 after every call.
 *
 * mec_chunk_signatures_device verifies `count` rows whose messages are already in device memory in ONE launch (shaped like
 * mec_sums_device): row i hashes d_base[offsets[i], + lens[i]) (any alignment), with prev + 64i the previous signature and
 * claimed + 64i the claimed one; kinds[i] is MEC_SIGV4_PAYLOAD (a chunk payload) or MEC_SIGV4_TRAILER (a trailer value, with
 * the '\n' readTrailers appends already in place).  verdicts[i] (host) is 1 when the claim equals the lowercase hex signature
 * byte for byte, else 0.  Returns MEC_OK once the verdicts are written (it waits for its work on cuda_stream); NULL arrays with
 * count > 0, negative offsets or lengths, an unknown kind or a head that does not fit are MEC_ERR_INVALID_ARGUMENT before any
 * device work.
 *
 * mec_encode_chunked is newSignV4ChunkedReader + Erasure.Encode of PutObject / PutObjectPart / PutObjectExtract: it de-frames the
 * aws-chunked `body` as s3ChunkedReader.Read does (cmd/streaming-signature-v4.go:264-442; only header bytes are read on the host),
 * checks every chunk's signature on the device, starting from the seed signature `seed` (64 lowercase hex bytes), and writes
 * mec_encode's part files of the decoded_len (x-amz-decoded-content-length) decoded bytes.  trailer != 0 reads the signed trailer
 * behind the final chunk as readTrailers does (:445-512) and returns its value as signed (with the '\n' readTrailers appends) in
 * trailer_out[0, min(trailer_cap, *trailer_len)); parsing its key:value lines and checking them against X-Amz-Trailer stay with
 * the caller.  Returns decoded_len, or the first error in stream order, per chunk: MEC_ERR_MALFORMED_ENCODING /
 * MEC_ERR_CHUNK_TOO_BIG (its header), MEC_ERR_INCOMPLETE_BODY (the body ends), MEC_ERR_SIGNATURE_MISMATCH, MEC_ERR_MALFORMED_ENCODING
 * (the CRLF behind the payload), MEC_ERR_OVERREAD (more payload than decoded_len); then MEC_ERR_INCOMPLETE_BODY for fewer payload
 * bytes than decoded_len.  After an error the part files are unspecified.  NULL or negative arguments, a seed that is not 64
 * lowercase hex bytes or a head that does not fit are MEC_ERR_INVALID_ARGUMENT, then MEC_ERR_WRITE_QUORUM, both before any device
 * work; so is an error in the first chunk's header.  "checksums" covers the decoded bytes. */
#define MEC_SIGV4_PAYLOAD 0
#define MEC_SIGV4_TRAILER 1
int mec_chunk_signatures_device(mec_codec* c, const uint8_t key[32], const char* date, const char* scope, const uint8_t* d_base,
                                const int64_t* offsets, const int64_t* lens, const uint8_t* prev, const uint8_t* claimed,
                                const int32_t* kinds, int64_t count, uint8_t* verdicts, void* cuda_stream);
int64_t mec_encode_chunked(mec_codec* c, const uint8_t* body, int64_t body_len, int64_t decoded_len, const uint8_t key[32],
                           const uint8_t seed[64], const char* date, const char* scope, int trailer, uint8_t* const* files,
                           int write_quorum, uint8_t* trailer_out, int64_t trailer_cap, int64_t* trailer_len);
/* mec_encode_chunked_sse is newSignV4ChunkedReader + EncryptRequest + Erasure.Encode, the PutObject / PutObjectPart of an encrypted
 * bucket (SSE-S3, SSE-KMS) with a streaming-signed body: mec_encode_chunked's de-framing and verdicts (sig_key as its `key`), then
 * mec_encode_sse of the decoded bytes with sse_key (the object key, or the part key) and nonce, in one pass of the encode pipeline.
 * On success the part files are byte-identical to mec_encode_sse's of the decoded bytes (sized for
 * mec_dare_encrypted_size(decoded_len)) and it returns decoded_len.  For any body it returns what mec_encode_chunked returns for that
 * body, in the same stream order; trailer mode returns the signed trailer value as mec_encode_chunked does.  Refusals:
 * mec_encode_chunked's, a NULL sse_key or nonce (MEC_ERR_INVALID_ARGUMENT) and a decoded_len no DARE stream holds, then
 * MEC_ERR_WRITE_QUORUM, all before any device work; so is an error in the first chunk's header.  After an error the part files are
 * unspecified.  An empty object verifies its final chunk (and trailer) rows and writes nothing.  "checksums" covers the decoded
 * plaintext, each byte once.  Both keys are zeroed on the device and the host before it returns.  At option "dare_chacha20" 2 the
 * packages are ChaCha20-Poly1305, as mec_encode_sse's. */
int64_t mec_encode_chunked_sse(mec_codec* c, const uint8_t* body, int64_t body_len, int64_t decoded_len, const uint8_t sig_key[32],
                               const uint8_t seed[64], const char* date, const char* scope, int trailer, const uint8_t sse_key[32],
                               const uint8_t nonce[12], uint8_t* const* files, int write_quorum, uint8_t* trailer_out,
                               int64_t trailer_cap, int64_t* trailer_len);

/* ---- shard-shaped low-level calls (keep Erasure.EncodeData / reedsolomon.Encoder shapes) ---- */
/* reedsolomon.Encoder.Encode: shards[0..k) in, shards[k..k+m) out, each shard_len bytes (host). */
int mec_rs_encode_shards(mec_codec* c, uint8_t* const* shards, int64_t shard_len);
/* reedsolomon.Encoder.Reconstruct / ReconstructData: shards[i] with present[i]==0 are rebuilt in
 * place (buffers must exist). */
int mec_rs_reconstruct_shards(mec_codec* c, uint8_t* const* shards, const uint8_t* present,
                              int64_t shard_len, int data_only);
/* hash.Hash one-shot for BitrotAlgorithm.New() == HighwayHash256(S) (cmd/bitrot.go:55-58): digests
 * of `count` equal-length messages laid out back to back (host). */
int mec_hh256_batch(mec_codec* c, const uint8_t* msgs, int64_t msg_len, int64_t count, uint8_t* digests);

/* erasureSelfTest + bitrotSelfTest (cmd/erasure-coding.go:149, cmd/bitrot.go:224) on the GPU. */
int mec_selftest(int device);

/* tuning knobs for benchmarks/tests (erasure blocks per CTA, loader, GF specialisation), and "dare_chacha20" (0, 1 or 2: which
 * DARE 2.0 AEADs the SSE calls open and seal, see above; any other value is MEC_ERR_INVALID_ARGUMENT and keeps the old one).
 * "jit": run-time specialisation of decode matrices / uncompiled (k, m) geometries with NVRTC, cached per process:
 *   -1 (default) a pattern that has been seen with 32 MiB of input is compiled on a background thread; calls that
 *      arrive before it is ready run the generic runtime-matrix kernel — no request ever waits for the compiler;
 *    1 compile (or wait for the background compile) inside the call — tests and benchmarks;  0 never specialise.
 * Compiled kernels are also kept on disk (MEC_JIT_CACHE_DIR, default $HOME/.cache/minio_b200, "off" disables), keyed by the kernel
 * sources, options and matrix: a restarted process loads the kernel of a pattern it has met before instead of recompiling.
 * "small_blocks": launches of at most this many erasure blocks run the latency form of the kernel (one CTA per block, hash warps
 *   decoupled from the GF warps: ~0.16 ms for a 1 MiB block instead of ~0.45 ms on an H100); -1 (default) = five per SM, 0 = never. */
int mec_set_option(mec_codec* c, const char* name, int64_t value);
/* Boundary counters (SURVEY §5 metrics row): name is one of "launches", "blocks_encoded", "blocks_read",
 * "shards_rebuilt", "corrupt_shards", "bytes_h2d", "bytes_d2h", "whole_hash_launches" (whole-file hash kernel launches), "jit_compiles", "jit_ms", "jit_disk_hits" (process-wide), "jit_launches",
 * "small_launches" (launches that took the latency form).  -1 for unknown names.
 * Kernel dispatch (which form of the fused kernel ran, for tests and diagnosis): "form_<f>" counts the launches of form f, one of
 *   small (latency kernel), fast3d, fast3d_auto, fast3d_semi, fast, fast_auto, aligned, aligned_auto, runtime, bytewise (the
 *   compile-time (k, m) kernels), dyn_aligned, dyn_runtime, dyn_bytewise (runtime matrix), jit (NVRTC-specialised);
 *   the last fused launch: "last_eb" (erasure blocks per CTA), "last_grid" (CTAs), "last_tma_mode" (0 byte-wise, 1 2-D boxes per
 *   row, 2 one tensor map per input, 3 runs of uniformly spaced inputs; -1 latency kernel), "last_rows3d" (one 3-D request per
 *   tile), "last_direct" (rows fetched straight into the hashed tile), "last_tiles3d" (tiles of a shard fetched in 3-D),
 *   "last_row_chunk" (runtime-matrix rows per pass: 0, 1, 2 for 1, 2, 4; -1 for a compile-time matrix); "num_sms".
 * Every ABI call is also wrapped in an NVTX range (visible in Nsight Systems) — the tracing hook of SURVEY §5. */
int64_t mec_get_stat(const mec_codec* c, const char* name);
/* Stops background kernel specialisation and waits for a compile in flight.  Call before the process exits (exit()
 * during an NVRTC compile lets libnvrtc's exit handlers run under the compiling thread); later calls of the library
 * keep working with the kernels already in the cache.  Also registered with atexit() after the first background compile. */
void mec_shutdown(void);
/* Queues, on the background compiler, the specialised kernels of every single-missing-data-shard pattern of the codec's geometry
 * (what a drive failure turns the next GETs and the heal into).  Returns the number of kernels queued; nothing blocks.  With the
 * on-disk cache this is a one-time cost per (k, m) and library version. */
int mec_jit_prewarm(mec_codec* c);
/* Build check of the run-time specialisation (no device needed): NVRTC-compiles the fused kernel for the r x k matrix `coef`
 * (align = S mod 16 of the inputs, eb = erasure blocks per CTA or 0, rows3d / hash_outputs as the engine would pass them)
 * without loading it.  Returns the cubin size, 0 when the compile fails (log in mec_last_error), -1 without libnvrtc. */
int64_t mec_jit_compile_check(int k, int r, const uint8_t* coef, int align, int eb, int rows3d, int hash_outputs);
/* number of kernels launched by this codec so far (bench.py's gpu_launches) */
int64_t mec_launch_count(const mec_codec* c);

#ifdef __cplusplus
}
#endif
#endif
