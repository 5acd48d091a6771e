// conc_bench.cc — the many-small-concurrent-requests regime (cmd/erasure-object.go:1371-1441: one Erasure per request, one block
// per loop iteration, thousands of request goroutines): T host threads each PUT (or degraded-GET) objects of a fixed size.
//   mode batcher : every PUT goes through ONE mec_batcher (cross-request coalescing into merged launches)
//   mode batcher_crc : the same PUTs, each also asking for its CRC32, CRC32C and CRC64NVME (mec_batcher_encode_crc); after the timed
//                  window every thread's last checksums are checked against a table CRC computed here on the host
//   mode batcher_sums : the same PUTs, each also asking for the object hashes of the mask SUMS (default 8 = MEC_SUM_MD5, the ETag;
//                  40 = MD5 | SHA-256) through mec_batcher_encode_sums; after the timed window every thread's last digests are checked
//                  against an MD5 written out here and the oracle's SHA-256
//   mode pool    : every thread picks a codec handle from a pool of P (no coalescing: one launch per call)
//   mode get     : degraded GETs (4 data drives offline) through the pool
//   mode bheal   : heals of one stale data drive (Erasure.Heal, the MRF / new-disk traffic) through ONE mec_batcher
//   mode heal    : the same heals, each a mec_heal_prefer call on a handle from the pool
//   mode bget_rot / bheal_rot : bget / bheal as MinIO lays objects out: thread t's object has its shard indices rotated by t % n over
//                  the drives (hashOrder, cmd/erasure-metadata-utils.go:178), and ONE physical drive (drive 0) is offline (GET) or
//                  stale (heal) — so the shard it held rotates from object to object: n erasure patterns in every round of requests
//   mode btranscode : moves of whole parts from RS(12,4) to the destination geometry DST="k2,m2" (default 6,2; decommission and
//                  rebalance, mec_batcher_transcode) through ONE transcode batcher (mec_batcher_new_transcode_ex); block sizes in bytes
//                  SRC_BS (source) and DST_BS (destination), default 1 MiB each (legacy 10 MiB-block parts: SRC_BS=10485760)
//   mode transcode : the same moves, each a mec_transcode call on the handle pair t % P (source and destination codec)
//   btranscode_rot / transcode_rot : as bget_rot, drive 0 offline and thread t's object rotated by t % n
//   mode btranscode_whole / transcode_whole (and their _rot forms): the same moves of parts written with the whole-file bitrot
//                  algorithm ALGO (1 = SHA256, 2 = HighwayHash256 (default), 4 = BLAKE2b512), their raw shard files and sums made
//                  once by mec_encode_whole: through ONE transcode batcher (mec_batcher_transcode_whole), or each a
//                  mec_transcode_whole call on the handle pair t % P (source codecs of that algorithm)
//                  (after the timed window every thread's out files are compared with a plain mec_encode on the destination geometry)
//   mode bget_mixed / bheal_mixed : GETs of whole objects / heals of one stale drive of legacy parts whose drives mix bitrot formats,
//                  through ONE mec_batcher (mec_batcher_decode_mixed / mec_batcher_heal_mixed): drives [0, HEALED) were already healed
//                  into HighwayHash256S frames (HEALED, default 8), the others hold raw shard files of the whole-file algorithm ALGO (as
//                  above) with sums made once by mec_encode_whole; a heal rebuilds drive HEALED (the next legacy drive; drive n - 1 when
//                  HEALED = n) from the others.  After the timed window every GET's bytes and every healed part file are checked.
//   mode get_mixed / heal_mixed : the same calls, each a mec_decode_mixed / mec_heal_mixed call on a handle from the pool
//   mode bverify / verify : VerifyFile of one object on one drive (the deep-scan heal's per-drive check): each call verifies drive
//                  t % n's shard file of the thread's object, written with ALGO (3 = HighwayHash256S frames; 1, 2, 4 = a raw shard file
//                  with its whole-file sum made once by mec_encode_whole), through ONE mec_batcher (mec_batcher_verify) or each a
//                  mec_bitrot_verify_parts call on a handle from the pool.  Every call must return MEC_OK with a clean result.
//   mode bsse_put / sse_put : encrypted PUTs (DARE 2.0, a key and nonce per thread) through ONE mec_batcher (mec_batcher_encode_sse)
//                  or each a mec_encode_sse call on a handle from the pool; after the timed window every thread's part files are
//                  compared with a mec_encode_sse of its object here
//   mode bsse_get / sse_get : degraded GETs (4 data drives offline) of whole encrypted objects through ONE mec_batcher
//                  (mec_batcher_decode_sse) or each a mec_decode_sse call on a handle from the pool
//   mode bsse_mixget : even threads GET encrypted objects, odd threads plain ones, through ONE mec_batcher (the two kinds share batches)
//                  (after the timed window every GET's bytes are compared with the object)
//   MIX=1        : the batcher of the b* modes is created with MEC_BATCHER_MIX_PATTERNS (reads of different patterns share batches)
//   mode cpu     : the C oracle's SIMD encode + HighwayHash on the calling thread (the reference's per-request CPU path)
// Prints one JSON line: aggregate GiB/s, calls/s, p50/p99 latency.  Buffers are pinned (mec_alloc_pinned_on) for the GPU modes.
// Build: g++ -O2 -std=c++17 tools/conc_bench.cc -o tools/conc_bench -Iinclude -Lminio_b200 -lminio_ec -Loracle -loracle -lpthread
#include <algorithm>
#include <execinfo.h>
#include <signal.h>
#include <unistd.h>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>
#include "minio_ec.h"
extern "C" void orc_encode_hash_blocks_st(int k, int m, int64_t bs, const uint8_t* src, int64_t nblocks, uint8_t* parity, uint8_t* digests);
extern "C" void orc_sha256(const uint8_t* p, size_t n, uint8_t out[32]);

// byte-at-a-time table CRC (reflected, init and xorout all ones): CRC32, CRC32C, CRC64NVME as Go's hash/crc32 and hash/crc64 give them
static uint64_t host_crc(const uint8_t* p, int64_t n, uint64_t poly, int bits) {
  uint64_t tab[256];
  for (int v = 0; v < 256; v++) {
    uint64_t c = static_cast<uint64_t>(v);
    for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ poly : c >> 1;
    tab[v] = c;
  }
  const uint64_t mask = bits == 64 ? ~0ull : (1ull << bits) - 1;
  uint64_t c = mask;
  for (int64_t i = 0; i < n; i++) c = tab[(c ^ p[i]) & 0xff] ^ (c >> 8);
  return c ^ mask;
}

// MD5 (RFC 1321), a byte-at-a-time host reference for the batcher_sums check
static void host_md5(const uint8_t* p, int64_t n, uint8_t out[16]) {
  static const uint32_t K[64] = {
      0xd76aa478, 0xe8c7b756, 0x242070db, 0xc1bdceee, 0xf57c0faf, 0x4787c62a, 0xa8304613, 0xfd469501, 0x698098d8, 0x8b44f7af, 0xffff5bb1,
      0x895cd7be, 0x6b901122, 0xfd987193, 0xa679438e, 0x49b40821, 0xf61e2562, 0xc040b340, 0x265e5a51, 0xe9b6c7aa, 0xd62f105d, 0x02441453,
      0xd8a1e681, 0xe7d3fbc8, 0x21e1cde6, 0xc33707d6, 0xf4d50d87, 0x455a14ed, 0xa9e3e905, 0xfcefa3f8, 0x676f02d9, 0x8d2a4c8a, 0xfffa3942,
      0x8771f681, 0x6d9d6122, 0xfde5380c, 0xa4beea44, 0x4bdecfa9, 0xf6bb4b60, 0xbebfbc70, 0x289b7ec6, 0xeaa127fa, 0xd4ef3085, 0x04881d05,
      0xd9d4d039, 0xe6db99e5, 0x1fa27cf8, 0xc4ac5665, 0xf4292244, 0x432aff97, 0xab9423a7, 0xfc93a039, 0x655b59c3, 0x8f0ccc92, 0xffeff47d,
      0x85845dd1, 0x6fa87e4f, 0xfe2ce6e0, 0xa3014314, 0x4e0811a1, 0xf7537e82, 0xbd3af235, 0x2ad7d2bb, 0xeb86d391};
  static const int R[16] = {7, 12, 17, 22, 5, 9, 14, 20, 4, 11, 16, 23, 6, 10, 15, 21};
  uint32_t h[4] = {0x67452301, 0xefcdab89, 0x98badcfe, 0x10325476};
  const int64_t nblk = (n + 8) / 64 + 1;  // message, 0x80, zeros, 8-byte length
  for (int64_t b = 0; b < nblk; b++) {
    uint32_t w[16] = {};
    for (int i = 0; i < 64; i++) {
      const int64_t pos = b * 64 + i;
      uint32_t v = pos < n ? p[pos] : pos == n ? 0x80 : 0;
      if (b == nblk - 1 && i >= 56) v = static_cast<uint8_t>(static_cast<uint64_t>(n) * 8 >> (8 * (i - 56)));
      w[i / 4] |= v << (8 * (i % 4));
    }
    uint32_t a = h[0], bb = h[1], c = h[2], d = h[3];
    for (int i = 0; i < 64; i++) {
      uint32_t f;
      int g;
      if (i < 16) { f = (bb & c) | (~bb & d); g = i; }
      else if (i < 32) { f = (d & bb) | (~d & c); g = (5 * i + 1) % 16; }
      else if (i < 48) { f = bb ^ c ^ d; g = (3 * i + 5) % 16; }
      else { f = c ^ (bb | ~d); g = (7 * i) % 16; }
      const uint32_t x = a + f + K[i] + w[g];
      const int r = R[(i / 16) * 4 + i % 4];
      a = d; d = c; c = bb;
      bb = bb + ((x << r) | (x >> (32 - r)));
    }
    h[0] += a; h[1] += bb; h[2] += c; h[3] += d;
  }
  for (int i = 0; i < 16; i++) out[i] = static_cast<uint8_t>(h[i / 4] >> (8 * (i % 4)));
}

static void on_segv(int sig) {
  void* bt[48];
  const int n = backtrace(bt, 48);
  fprintf(stderr, "signal %d, backtrace:\n", sig);
  backtrace_symbols_fd(bt, n, 2);
  _exit(139);
}

int main(int argc, char** argv) {
  signal(SIGSEGV, on_segv);
  signal(SIGABRT, on_segv);
  std::string mode = argc > 1 ? argv[1] : "batcher";
  const bool rot = mode == "bget_rot" || mode == "bheal_rot" || mode == "btranscode_rot" || mode == "transcode_rot" ||
                   mode == "btranscode_whole_rot" || mode == "transcode_whole_rot";
  if (rot) mode.resize(mode.size() - 4);
  const std::string mode_name = rot ? mode + "_rot" : mode;
  const int bflags = getenv("MIX") && atoi(getenv("MIX")) ? MEC_BATCHER_MIX_PATTERNS : 0;
  const int T = argc > 2 ? atoi(argv[2]) : 256;
  // object size: MiB, or KiB with a 'k' suffix (objects smaller than one erasure block: "256k")
  const std::string osz = argc > 3 ? argv[3] : "1";
  const int64_t osize = (!osz.empty() && (osz.back() == 'k' || osz.back() == 'K')) ? atoll(osz.c_str()) << 10 : atoll(osz.c_str()) << 20;
  const int calls_per_thread = argc > 4 ? atoi(argv[4]) : 32;
  const int P = argc > 5 ? atoi(argv[5]) : 8;
  const int device = argc > 6 ? atoi(argv[6]) : 0;
  const int k = 12, m = 4, n = k + m;
  const bool whole = mode == "btranscode_whole" || mode == "transcode_whole";
  const bool bmove = mode == "btranscode" || mode == "btranscode_whole";  // through the transcode batcher
  const bool move = bmove || mode == "transcode" || mode == "transcode_whole";
  const int walgo = getenv("ALGO") ? atoi(getenv("ALGO")) : MEC_HIGHWAYHASH256;
  const bool bmixed = mode == "bget_mixed" || mode == "bheal_mixed";  // through the batcher
  const bool mixed = bmixed || mode == "get_mixed" || mode == "heal_mixed";
  const bool mixed_get = mode == "bget_mixed" || mode == "get_mixed";
  const int healed = getenv("HEALED") ? std::max(0, std::min(k + m, atoi(getenv("HEALED")))) : 8;
  const int mixed_stale = std::min(healed, k + m - 1);
  const bool bverify = mode == "bverify", verify = bverify || mode == "verify";
  const bool vwhole = verify && walgo != MEC_HIGHWAYHASH256S;
  const int64_t bs = move && getenv("SRC_BS") ? atoll(getenv("SRC_BS")) : 1 << 20;
  const int64_t bs2 = move && getenv("DST_BS") ? atoll(getenv("DST_BS")) : 1 << 20;
  const bool gpu = mode != "cpu";
  const bool bsse = mode == "bsse_put" || mode == "bsse_get" || mode == "bsse_mixget";  // through the batcher
  const bool sse = bsse || mode == "sse_put" || mode == "sse_get";
  const bool sse_put = mode == "bsse_put" || mode == "sse_put";
  mec_codec* probe = nullptr;
  mec_codec_new(k, m, bs, MEC_HIGHWAYHASH256S, device, &probe);
  // an encrypted object is stored as its DARE 2.0 stream: part files are sized for that
  const int64_t esize = sse ? mec_dare_encrypted_size(osize) : osize;
  const int64_t S = mec_shard_size(probe), fsz = mec_bitrot_shard_file_size(mec_shard_file_size(probe, esize), S, MEC_HIGHWAYHASH256S);
  const int64_t nb = (esize + bs - 1) / bs;
  // thread t's key and nonce (encrypted modes; bsse_mixget: even threads)
  auto sse_key = [](int t, uint8_t* key, uint8_t* nonce) {
    for (int i = 0; i < 32; i++) key[i] = static_cast<uint8_t>(t * 131 + i * 7 + 1);
    for (int i = 0; i < 12; i++) nonce[i] = static_cast<uint8_t>(t * 17 + i * 29 + 3);
  };
  auto encrypted = [&](int t) { return sse && (mode != "bsse_mixget" || t % 2 == 0); };
  int k2 = 6, m2 = 2;
  if (const char* e = getenv("DST")) sscanf(e, "%d,%d", &k2, &m2);
  const int n2 = k2 + m2;
  mec_codec* probe2 = nullptr;
  mec_codec_new(k2, m2, bs2, MEC_HIGHWAYHASH256S, device, &probe2);
  const int64_t fsz2 = mec_bitrot_shard_file_size(mec_shard_file_size(probe2, osize), mec_shard_size(probe2), MEC_HIGHWAYHASH256S);
  if (gpu) mec_bind_thread_to_device(device);
  auto alloc = [&](size_t b) -> uint8_t* { return gpu ? static_cast<uint8_t*>(mec_alloc_pinned_on(device, b)) : static_cast<uint8_t*>(malloc(b)); };
  // per-thread buffers: object, 16 part files, digests, destination, the healed part file
  const int sums_mask = getenv("SUMS") ? atoi(getenv("SUMS")) : MEC_SUM_MD5;
  struct TB { uint8_t* obj; std::vector<uint8_t*> files; uint8_t* dd; uint8_t* dst; uint8_t* parity; uint8_t* healed; uint64_t crc[3];
              uint8_t sums[MEC_SUM_BYTES];
              std::vector<uint8_t> wsums;  // whole-file and mixed modes: the expected digest of every source shard file, n x 64
              std::vector<uint8_t*> wfiles;  // mixed modes: every drive's raw shard file of the whole-file algorithm
              std::vector<uint8_t*> outs;  // outs: the destination part files of the transcode modes
              uint8_t key[32], nonce[12]; };  // outs: the destination part files of the transcode modes
  std::vector<TB> tb(T);
  uint8_t* arena = alloc(static_cast<size_t>(T) * (osize * 2 + (n + 1) * fsz + nb * n * 32 + nb * m * S + 4096 * 25));
  if (!arena) { fprintf(stderr, "allocation failed\n"); return 1; }
  uint8_t* p = arena;
  auto take = [&](size_t b) { uint8_t* r = p; p += (b + 4095) / 4096 * 4096; return r; };
  uint64_t x = 88172645463325252ull;
  for (int t = 0; t < T; t++) {
    tb[t].obj = take(osize);
    for (int64_t i = 0; i < osize / 8; i++) { x ^= x << 13; x ^= x >> 7; x ^= x << 17; reinterpret_cast<uint64_t*>(tb[t].obj)[i] = x; }
    for (int i = 0; i < n; i++) tb[t].files.push_back(take(fsz));
    tb[t].dd = take(nb * n * 32);
    tb[t].dst = take(osize);
    tb[t].parity = take(nb * m * S);
    tb[t].healed = take(fsz);
    if (mixed || vwhole)
      for (int i = 0; i < n; i++) {
        tb[t].wfiles.push_back(alloc(static_cast<size_t>(std::max<int64_t>(1, mec_shard_file_size(probe, osize)))));
        if (!tb[t].wfiles.back()) { fprintf(stderr, "allocation failed\n"); return 1; }
      }
    if (move)
      for (int i = 0; i < n2; i++) {
        tb[t].outs.push_back(alloc(static_cast<size_t>(fsz2)));
        if (!tb[t].outs.back()) { fprintf(stderr, "allocation failed\n"); return 1; }
      }
  }
  mec_batcher* bat = nullptr;
  std::vector<mec_codec*> pool, pool2;
  if (mode == "batcher" || mode == "batcher_crc" || mode == "batcher_sums") {
    int rc = mec_batcher_new_ex(k, m, bs, device, getenv("MAX_BATCH") ? atoll(getenv("MAX_BATCH")) : 512, getenv("MAX_WAIT_US") ? atoi(getenv("MAX_WAIT_US")) : 100,
                                bflags, &bat);
    if (rc) { fprintf(stderr, "batcher: %d %s\n", rc, mec_last_error()); return 1; }
  } else if (gpu && mode != "bget" && mode != "bheal" && !bmove && !bmixed && !bverify && !bsse) {
    for (int i = 0; i < P; i++) { mec_codec* c = nullptr; mec_codec_new(k, m, bs, whole ? walgo : MEC_HIGHWAYHASH256S, device, &c); if (getenv("POOL_JIT")) mec_set_option(c, "jit", 1); pool.push_back(c); }
  }
  if (mode == "bget" || mode == "bheal") {  // coalesced GETs / heals: part files through a temporary handle, then everything goes through the batcher
    mec_codec* c0 = nullptr; mec_codec_new(k, m, bs, MEC_HIGHWAYHASH256S, device, &c0);
    for (int t = 0; t < T; t++) {
      std::vector<uint8_t*> f(tb[t].files);
      if (mec_encode(c0, tb[t].obj, osize, f.data(), k) != osize) { fprintf(stderr, "prep encode failed\n"); return 1; }
    }
    mec_codec_free(c0);
    int rc = mec_batcher_new_ex(k, m, bs, device, getenv("MAX_BATCH") ? atoll(getenv("MAX_BATCH")) : 512, getenv("MAX_WAIT_US") ? atoi(getenv("MAX_WAIT_US")) : 100,
                                bflags, &bat);
    if (rc) { fprintf(stderr, "batcher: %d\n", rc); return 1; }
  }
  if (sse) {  // keys; the stored parts of the GET modes through a temporary handle; the batcher of the bsse_* modes
    mec_codec* c0 = nullptr; mec_codec_new(k, m, bs, MEC_HIGHWAYHASH256S, device, &c0);
    for (int t = 0; t < T; t++) {
      sse_key(t, tb[t].key, tb[t].nonce);
      if (sse_put) continue;
      std::vector<uint8_t*> f(tb[t].files);
      const int64_t rc = encrypted(t) ? mec_encode_sse(c0, tb[t].obj, osize, tb[t].key, tb[t].nonce, f.data(), k)
                                      : mec_encode(c0, tb[t].obj, osize, f.data(), k);
      if (rc != osize) { fprintf(stderr, "prep encode failed\n"); return 1; }
    }
    mec_codec_free(c0);
    if (bsse) {
      int rc = mec_batcher_new_ex(k, m, bs, device, getenv("MAX_BATCH") ? atoll(getenv("MAX_BATCH")) : 512,
                                  getenv("MAX_WAIT_US") ? atoi(getenv("MAX_WAIT_US")) : 100, bflags, &bat);
      if (rc) { fprintf(stderr, "batcher: %d\n", rc); return 1; }
    }
  }
  if (mixed) {  // both formats of every part through temporary handles; the batcher of the b*_mixed modes
    mec_codec* cs = nullptr;
    mec_codec* cw = nullptr;
    mec_codec_new(k, m, bs, MEC_HIGHWAYHASH256S, device, &cs);
    mec_codec_new(k, m, bs, walgo, device, &cw);
    for (int t = 0; t < T; t++) {
      std::vector<uint8_t*> f(tb[t].files), w(tb[t].wfiles);
      tb[t].wsums.assign(static_cast<size_t>(n) * 64, 0);
      if (mec_encode(cs, tb[t].obj, osize, f.data(), k) != osize || mec_encode_whole(cw, tb[t].obj, osize, w.data(), tb[t].wsums.data(), k) != osize) {
        fprintf(stderr, "prep encode failed\n");
        return 1;
      }
    }
    mec_codec_free(cs);
    mec_codec_free(cw);
    if (bmixed) {
      int rc = mec_batcher_new_ex(k, m, bs, device, getenv("MAX_BATCH") ? atoll(getenv("MAX_BATCH")) : 512,
                                  getenv("MAX_WAIT_US") ? atoi(getenv("MAX_WAIT_US")) : 100, bflags, &bat);
      if (rc) { fprintf(stderr, "batcher: %d\n", rc); return 1; }
    }
  }
  if (verify) {  // every drive's shard file in the format of ALGO through temporary handles; the batcher of bverify
    mec_codec* c0 = nullptr;
    mec_codec_new(k, m, bs, walgo, device, &c0);
    for (int t = 0; t < T; t++) {
      std::vector<uint8_t*> f(vwhole ? tb[t].wfiles : tb[t].files);
      tb[t].wsums.assign(static_cast<size_t>(n) * 64, 0);
      const int64_t rc = vwhole ? mec_encode_whole(c0, tb[t].obj, osize, f.data(), tb[t].wsums.data(), k) : mec_encode(c0, tb[t].obj, osize, f.data(), k);
      if (rc != osize) { fprintf(stderr, "prep encode failed\n"); return 1; }
    }
    mec_codec_free(c0);
    if (bverify) {
      int rc = mec_batcher_new_ex(k, m, bs, device, getenv("MAX_BATCH") ? atoll(getenv("MAX_BATCH")) : 512,
                                  getenv("MAX_WAIT_US") ? atoi(getenv("MAX_WAIT_US")) : 100, bflags, &bat);
      if (rc) { fprintf(stderr, "batcher: %d\n", rc); return 1; }
    }
  }
  if (move) {  // source part files through a temporary handle; the transcode batcher, or the pool's destination handles
    mec_codec* c0 = nullptr; mec_codec_new(k, m, bs, whole ? walgo : MEC_HIGHWAYHASH256S, device, &c0);
    for (int t = 0; t < T; t++) {
      std::vector<uint8_t*> f(tb[t].files);
      tb[t].wsums.assign(static_cast<size_t>(n) * 64, 0);
      const int64_t rc = whole ? mec_encode_whole(c0, tb[t].obj, osize, f.data(), tb[t].wsums.data(), k) : mec_encode(c0, tb[t].obj, osize, f.data(), k);
      if (rc != osize) { fprintf(stderr, "prep encode failed\n"); return 1; }
    }
    mec_codec_free(c0);
    if (bmove) {
      int rc = mec_batcher_new_transcode_ex(k, m, bs, k2, m2, bs2, device, getenv("MAX_BATCH") ? atoll(getenv("MAX_BATCH")) : 512,
                                            getenv("MAX_WAIT_US") ? atoi(getenv("MAX_WAIT_US")) : 100, bflags, &bat);
      if (rc) { fprintf(stderr, "transcode batcher: %d %s\n", rc, mec_last_error()); return 1; }
    } else {
      for (int i = 0; i < P; i++) { mec_codec* c = nullptr; mec_codec_new(k2, m2, bs2, MEC_HIGHWAYHASH256S, device, &c); pool2.push_back(c); }
    }
  }
  if (mode == "get" || mode == "heal") {  // every thread's part files must exist first
    for (int t = 0; t < T; t++) {
      std::vector<uint8_t*> f(tb[t].files);
      if (mec_encode(pool[t % P], tb[t].obj, osize, f.data(), k) != osize) { fprintf(stderr, "prep encode failed\n"); return 1; }
    }
  }
  std::atomic<int> ready{0}, go{0};
  std::atomic<int64_t> errors{0};
  std::vector<std::vector<double>> lat(T);
  // the shard index physical drive 0 holds for thread t's object: its rotation is t % n (the _rot modes), none otherwise
  auto drive0_shard = [&](int t) { return rot ? (n - t % n) % n : 0; };
  auto one_call = [&](int t) -> int64_t {
    TB& b = tb[t];
    if (mode == "batcher") return mec_batcher_encode_sg(bat, b.obj, osize, b.files.data(), b.dd, k + 1);
    if (mode == "batcher_crc") return mec_batcher_encode_crc(bat, b.obj, osize, b.files.data(), b.dd, k + 1, MEC_CRC32 | MEC_CRC32C | MEC_CRC64NVME, b.crc);
    if (mode == "batcher_sums") return mec_batcher_encode_sums(bat, b.obj, osize, b.files.data(), b.dd, k + 1, sums_mask, nullptr, b.sums);
    if (mode == "pool") return mec_encode_sg(pool[t % P], b.obj, osize, b.files.data(), b.dd, k + 1);
    if (mode == "bget") {
      const uint8_t* f[64];
      for (int i = 0; i < n; i++) f[i] = (rot ? i == drive0_shard(t) : i < 4) ? nullptr : b.files[i];
      int hint = 0;
      return mec_batcher_decode(bat, f, 0, osize, osize, b.dst, &hint);
    }
    if (mode == "get") {
      const uint8_t* f[64];
      for (int i = 0; i < n; i++) f[i] = i < 4 ? nullptr : b.files[i];
      int hint = 0;
      return mec_decode(pool[t % P], f, 0, osize, osize, b.dst, &hint);
    }
    if (mode == "bheal" || mode == "heal") {  // drive 0 is stale: its part file is rebuilt from the first k of the others
      const uint8_t* f[64];
      uint8_t* o[64] = {};
      uint8_t bad[64];
      const int st = drive0_shard(t);
      for (int i = 0; i < n; i++) f[i] = i == st ? nullptr : b.files[i];
      o[st] = b.healed;
      const int rc = mode == "bheal" ? mec_batcher_heal(bat, f, nullptr, osize, o, bad) : mec_heal_prefer(pool[t % P], f, nullptr, osize, o, bad);
      return rc == MEC_OK ? osize : rc;
    }
    if (sse_put) {
      if (mode == "bsse_put") return mec_batcher_encode_sse(bat, b.obj, osize, b.key, b.nonce, b.files.data(), k + 1);
      return mec_encode_sse(pool[t % P], b.obj, osize, b.key, b.nonce, b.files.data(), k + 1);
    }
    if (sse) {  // 4 data drives offline
      const uint8_t* f[64];
      for (int i = 0; i < n; i++) f[i] = i < 4 ? nullptr : b.files[i];
      int hint = 0;
      if (!encrypted(t)) return mec_batcher_decode(bat, f, 0, osize, osize, b.dst, &hint);
      if (bsse) return mec_batcher_decode_sse(bat, f, nullptr, 0, osize, esize, b.key, b.dst, &hint);
      return mec_decode_sse(pool[t % P], f, nullptr, 0, osize, esize, b.key, b.dst, &hint);
    }
    if (mixed) {  // drives [0, healed) stream, the others are raw shard files; a heal rebuilds drive mixed_stale
      const uint8_t* f[64];
      uint8_t* o[64] = {};
      uint8_t bad[64];
      int al[64];
      for (int i = 0; i < n; i++) {
        al[i] = i < healed ? MEC_HIGHWAYHASH256S : walgo;
        f[i] = i < healed ? b.files[i] : b.wfiles[i];
      }
      int hint = 0;
      if (mode == "bget_mixed") return mec_batcher_decode_mixed(bat, al, f, b.wsums.data(), nullptr, 0, osize, osize, b.dst, &hint);
      if (mode == "get_mixed") return mec_decode_mixed(pool[t % P], al, f, b.wsums.data(), nullptr, 0, osize, osize, b.dst, &hint);
      f[mixed_stale] = nullptr;
      o[mixed_stale] = b.healed;
      const int rc = bmixed ? mec_batcher_heal_mixed(bat, al, f, b.wsums.data(), nullptr, osize, o, bad)
                            : mec_heal_mixed(pool[t % P], al, f, b.wsums.data(), nullptr, osize, o, bad);
      return rc == MEC_OK ? osize : rc;
    }
    if (verify) {  // one part: drive t % n's shard file as stored, its length, ShardFileSize(part.Size) and the whole-file sum
      const int i = t % n;
      const int algo = walgo;
      const uint8_t* f = vwhole ? b.wfiles[i] : b.files[i];
      const int64_t sfs = mec_shard_file_size(probe, osize);
      const int64_t flen = vwhole ? sfs : fsz;
      int res = -1;
      const int rc = bverify ? mec_batcher_verify(bat, 1, &algo, &f, &flen, &sfs, b.wsums.data() + i * 64, &res)
                             : mec_bitrot_verify_parts(pool[t % P], 1, &algo, &f, &flen, &sfs, b.wsums.data() + i * 64, &res);
      return rc == MEC_OK && res == MEC_OK ? osize : rc ? rc : res;
    }
    if (move) {  // drive 0 offline in the _rot modes
      const uint8_t* f[64];
      for (int i = 0; i < n; i++) f[i] = rot && i == drive0_shard(t) ? nullptr : b.files[i];
      int hint = 0;
      if (mode == "btranscode_whole") return mec_batcher_transcode_whole(bat, walgo, f, b.wsums.data(), nullptr, osize, b.outs.data(), k2, &hint);
      if (mode == "transcode_whole")
        return mec_transcode_whole(pool[t % P], f, b.wsums.data(), nullptr, osize, pool2[t % P], b.outs.data(), k2, &hint);
      return mode == "btranscode" ? mec_batcher_transcode(bat, f, nullptr, osize, b.outs.data(), k2, &hint)
                                  : mec_transcode(pool[t % P], f, nullptr, osize, pool2[t % P], b.outs.data(), k2, &hint);
    }
    orc_encode_hash_blocks_st(k, m, bs, b.obj, nb, b.parity, b.dd);
    return osize;
  };
  std::vector<std::thread> th;
  for (int t = 0; t < T; t++)
    th.emplace_back([&, t] {
      for (int w = 0; w < 2; w++) if (one_call(t) != osize) errors++;   // warm-up
      ready++;
      while (!go.load()) std::this_thread::yield();
      lat[t].reserve(calls_per_thread);
      for (int i = 0; i < calls_per_thread; i++) {
        const auto t0 = std::chrono::steady_clock::now();
        if (one_call(t) != osize) errors++;
        lat[t].push_back(std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count());
      }
    });
  while (ready.load() < T) std::this_thread::yield();
  const auto t0 = std::chrono::steady_clock::now();
  go = 1;
  for (auto& t : th) t.join();
  const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  if (mode == "bheal" || mode == "heal")  // every healed part file equals the drive's original one
    for (int t = 0; t < T; t++)
      if (memcmp(tb[t].healed, tb[t].files[drive0_shard(t)], static_cast<size_t>(fsz)) != 0) errors++;
  if (mixed)  // every GET's bytes equal the object, every healed part file the drive's streaming image
    for (int t = 0; t < T; t++)
      if (mixed_get ? memcmp(tb[t].dst, tb[t].obj, static_cast<size_t>(osize)) != 0
                    : memcmp(tb[t].healed, tb[t].files[mixed_stale], static_cast<size_t>(fsz)) != 0)
        errors++;
  if (sse_put) {  // every thread's part files equal a mec_encode_sse of its object with its key and nonce
    std::vector<uint8_t*> want(n);
    for (int i = 0; i < n; i++) want[i] = static_cast<uint8_t*>(malloc(static_cast<size_t>(fsz)));
    for (int t = 0; t < T; t++) {
      if (mec_encode_sse(probe, tb[t].obj, osize, tb[t].key, tb[t].nonce, want.data(), k) != osize) { errors++; continue; }
      for (int i = 0; i < n; i++)
        if (memcmp(tb[t].files[i], want[i], static_cast<size_t>(fsz)) != 0) errors++;
    }
    for (auto w : want) free(w);
  } else if (sse) {  // every GET's bytes equal the object
    for (int t = 0; t < T; t++)
      if (memcmp(tb[t].dst, tb[t].obj, static_cast<size_t>(osize)) != 0) errors++;
  }
  if (move) {  // every destination part file equals what a plain mec_encode of the destination geometry writes
    std::vector<uint8_t*> want(n2);
    for (int i = 0; i < n2; i++) want[i] = static_cast<uint8_t*>(malloc(static_cast<size_t>(fsz2)));
    for (int t = 0; t < T; t++) {
      if (mec_encode(probe2, tb[t].obj, osize, want.data(), k2) != osize) { errors++; continue; }
      for (int i = 0; i < n2; i++)
        if (memcmp(tb[t].outs[i], want[i], static_cast<size_t>(fsz2)) != 0) errors++;
    }
    for (auto w : want) free(w);
  }
  if (mode == "batcher_crc")  // every thread's object checksums equal the host's
    for (int t = 0; t < T; t++)
      if (tb[t].crc[0] != host_crc(tb[t].obj, osize, 0xEDB88320ull, 32) || tb[t].crc[1] != host_crc(tb[t].obj, osize, 0x82F63B78ull, 32) ||
          tb[t].crc[2] != host_crc(tb[t].obj, osize, 0x9A6C9329AC4BC9B5ull, 64))
        errors++;
  if (mode == "batcher_sums")  // every thread's digests equal the host's
    for (int t = 0; t < T; t++) {
      uint8_t want[32];
      if (sums_mask & MEC_SUM_MD5) { host_md5(tb[t].obj, osize, want); if (memcmp(tb[t].sums, want, 16)) errors++; }
      if (sums_mask & MEC_SUM_SHA256) { orc_sha256(tb[t].obj, static_cast<size_t>(osize), want); if (memcmp(tb[t].sums + 64, want, 32)) errors++; }
    }
  std::vector<double> all;
  for (auto& v : lat) all.insert(all.end(), v.begin(), v.end());
  std::sort(all.begin(), all.end());
  const double total = static_cast<double>(T) * calls_per_thread * osize;
  printf("{\"mode\": \"%s\", \"threads\": %d, \"object_MiB\": %lld, \"object_bytes\": %lld, \"calls\": %zu, \"seconds\": %.4f, \"GiB_per_s\": %.2f, \"calls_per_s\": %.0f, "
         "\"p50_us\": %.0f, \"p99_us\": %.0f, \"errors\": %lld",
         mode_name.c_str(), T, static_cast<long long>(osize >> 20), static_cast<long long>(osize), all.size(), sec, total / sec / (1 << 30), all.size() / sec, all[all.size() / 2],
         all[static_cast<size_t>(all.size() * 0.99)], static_cast<long long>(errors.load()));
  if (mode == "batcher_crc") printf(", \"crc_requests\": %lld", static_cast<long long>(mec_batcher_stat(bat, "crc_requests")));
  if (mode == "batcher_sums")
    printf(", \"sums_mask\": %d, \"sum_requests\": %lld", sums_mask, static_cast<long long>(mec_batcher_stat(bat, "sum_requests")));
  if (bat) printf(", \"mix\": %d, \"batches\": %lld, \"blocks_per_batch\": %.1f, \"launches\": %lld, \"patterns\": %lld, \"mixed_batches\": %lld",
                  bflags ? 1 : 0, static_cast<long long>(mec_batcher_stat(bat, "batches")),
                  static_cast<double>(mec_batcher_stat(bat, "blocks")) / std::max<int64_t>(1, mec_batcher_stat(bat, "batches")),
                  static_cast<long long>(mec_batcher_stat(bat, "launches")), static_cast<long long>(mec_batcher_stat(bat, "patterns")),
                  static_cast<long long>(mec_batcher_stat(bat, "mixed_batches")));
  if (bat && getenv("MEC_BATCHER_TRACE"))
    printf(", \"worker_us\": {\"submit\": %lld, \"sync\": %lld, \"finish\": %lld, \"idle\": %lld}, \"stream_us\": {\"stage\": %lld, \"kernel\": %lld, \"scatter\": %lld}",
           (long long)mec_batcher_stat(bat, "us_submit"), (long long)mec_batcher_stat(bat, "us_sync"), (long long)mec_batcher_stat(bat, "us_finish"),
           (long long)mec_batcher_stat(bat, "us_idle"), (long long)mec_batcher_stat(bat, "us_stage"), (long long)mec_batcher_stat(bat, "us_kernel"),
           (long long)mec_batcher_stat(bat, "us_scatter"));
  if (move) printf(", \"dst\": \"%d,%d\", \"src_block_size\": %lld, \"dst_block_size\": %lld", k2, m2, static_cast<long long>(bs),
                  static_cast<long long>(bs2));
  if (whole || mixed || verify) printf(", \"algo\": %d", walgo);
  if (bverify)
    printf(", \"verifies\": %lld, \"verifies_serial\": %lld, \"whole_hash_launches\": %lld", static_cast<long long>(mec_batcher_stat(bat, "verifies")),
           static_cast<long long>(mec_batcher_stat(bat, "verifies_serial")), static_cast<long long>(mec_batcher_stat(bat, "whole_hash_launches")));
  if (mixed) printf(", \"healed\": %d", healed);
  if (bsse)
    printf(", \"sse_puts\": %lld, \"sse_gets\": %lld, \"sse_serial\": %lld, \"redone\": %lld", static_cast<long long>(mec_batcher_stat(bat, "sse_puts")),
           static_cast<long long>(mec_batcher_stat(bat, "sse_gets")), static_cast<long long>(mec_batcher_stat(bat, "sse_serial")),
           static_cast<long long>(mec_batcher_stat(bat, "redone")));
  if (bmixed)
    printf(", \"reads_whole\": %lld, \"reads_whole_serial\": %lld, \"redone\": %lld, \"whole_hash_launches\": %lld",
           static_cast<long long>(mec_batcher_stat(bat, "reads_whole")), static_cast<long long>(mec_batcher_stat(bat, "reads_whole_serial")),
           static_cast<long long>(mec_batcher_stat(bat, "redone")), static_cast<long long>(mec_batcher_stat(bat, "whole_hash_launches")));
  if (mode == "btranscode")
    printf(", \"transcodes\": %lld, \"transcodes_serial\": %lld, \"redone\": %lld", static_cast<long long>(mec_batcher_stat(bat, "transcodes")),
           static_cast<long long>(mec_batcher_stat(bat, "transcodes_serial")), static_cast<long long>(mec_batcher_stat(bat, "redone")));
  if (mode == "btranscode_whole")
    printf(", \"transcodes_whole\": %lld, \"transcodes_whole_serial\": %lld, \"redone\": %lld, \"whole_hash_launches\": %lld",
           static_cast<long long>(mec_batcher_stat(bat, "transcodes_whole")), static_cast<long long>(mec_batcher_stat(bat, "transcodes_whole_serial")),
           static_cast<long long>(mec_batcher_stat(bat, "redone")), static_cast<long long>(mec_batcher_stat(bat, "whole_hash_launches")));
  if (mode == "pool" || mode == "get" || mode == "heal" || mode == "transcode" || mode == "transcode_whole" || mode == "get_mixed" ||
      mode == "heal_mixed" || mode == "verify" || mode == "sse_put" || mode == "sse_get")
    printf(", \"pool\": %d", P);
  printf("}\n");
  if (bat) mec_batcher_free(bat);
  for (auto c : pool) mec_codec_free(c);
  for (auto c : pool2) mec_codec_free(c);
  mec_codec_free(probe);
  mec_codec_free(probe2);
  mec_shutdown();  // no NVRTC compile may be in flight when the C runtime runs its exit handlers (a degraded-GET pattern warms up during the run)
  return errors.load() ? 2 : 0;
}
