"""Every form of the throughput kernel at the launch shapes that select it, every erasure block against the CPU oracle.

Engine::launch_fused picks the kernel from the launch size and the shard geometry, and the host-buffer entry points only ever make
launches small enough for the latency kernel or the eb 1-3 runtime instantiation.  The forms a large device-resident encode or
reconstruct runs are therefore driven here through mec_encode_blocks_device / mec_reconstruct_device at shapes chosen to select
them: each test asserts from the "form_*" / "last_*" dispatch counters that exactly the intended form ran, with the intended CTA
shape and 3-D tiling, and compares the parity (or rebuilt shards) and the digests of EVERY block with the oracle.  Parity rows are
written at a pitch wider than the shard and pre-filled, so a store past the end of a shard shows up in the guard bytes.

Shards of about 3 KiB (12-17 tiles of 256 bytes) keep the launches small; the options eb = 4 and grid_mult = 1 (one CTA per SM)
then give every CTA two or three groups of four blocks, the last group holding a single block.  Shard lengths sit at the edges of
the 3-D fetch: one or two per-row fallback tiles at the end of a shard, and full or partial last tiles.
"""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
MiB = 1 << 20
TILE = 256
FILL = 0xA5          # parity, digest and rebuilt-shard buffers are pre-filled with this byte
GUARD = 32           # parity rows are this much wider than round_up(S, 16)
FORMS = ("small", "fast3d", "fast3d_auto", "fast3d_semi", "fast", "fast_auto", "aligned", "aligned_auto", "runtime", "bytewise",
         "dyn_aligned", "dyn_runtime", "dyn_bytewise", "jit")
TMA_BYTEWISE, TMA_BLOCKS2D, TMA_PER_INPUT, TMA_RUNS = 0, 1, 2, 3    # LoaderMode (ec_kernel.cuh)
ROW_CHUNK = {1: 0, 2: 1, 3: 2, 4: 2}                                  # runtime-matrix row chunk index for r outputs


@pytest.fixture(scope="module")
def mb():
    import minio_b200
    assert minio_b200.device_count() > 0, "no CUDA device"
    return minio_b200


@pytest.fixture(scope="module")
def num_sms(mb):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture
def jit_cache(tmp_path, monkeypatch):
    """NVRTC-specialised kernels are compiled into (and loaded from) a directory of this test only."""
    monkeypatch.setenv("MEC_JIT_CACHE_DIR", str(tmp_path))


def round_up(x, a):
    return (x + a - 1) // a * a


def ceil_div(a, b):
    return -(-a // b)


def bs_for(k, S):
    """A block size that is a multiple of 16 (so TMA may fetch it) and whose shards are S bytes: ceil(bs / k) == S."""
    bs = k * S // 16 * 16
    assert bs > 0 and ceil_div(bs, k) == S, f"no 16-byte multiple block size has {k} shards of {S} bytes"
    return bs


def bs_unaligned(k, S):
    """The largest block size that is NOT a multiple of 16 and has shards of S bytes: only the byte-wise loader can fetch it."""
    bs = k * S
    while bs % 16 == 0:
        bs -= 1
    assert ceil_div(bs, k) == S
    return bs


def form_counts(c):
    got = {f: c.stat("form_" + f) for f in FORMS}
    assert min(got.values()) >= 0, got    # -1: the library does not know a form name
    return got


def form_delta(before, after):
    return {f: after[f] - before[f] for f in FORMS if after[f] != before[f]}


def last_launch(c):
    return {f: c.stat(f) for f in ("last_eb", "last_grid", "last_tma_mode", "last_rows3d", "last_direct", "last_tiles3d",
                                   "last_row_chunk", "num_sms")}


def oracle_blocks(oracle, k, m, bs, src):
    """Parity [nblocks, m, S] and the digests of all k + m shards [nblocks, k + m, 32] of every full block of `src`, from the
    oracle's multi-threaded encode + hash; checked against the scalar Split + Encode and HighwayHash on the first and last block
    of `src`."""
    S = ceil_div(bs, k)
    assert (k - 1) * S < bs, "the oracle's block encoder pads only the last data shard"
    nblocks = src.size // bs
    par = np.empty((nblocks, m, S), dtype=np.uint8)
    dig = np.empty((nblocks, k + m, 32), dtype=np.uint8)
    oracle.lib().orc_encode_hash_blocks_mt(k, m, bs, src.ctypes.data, nblocks, par.ctypes.data, dig.ctypes.data,
                                           len(os.sched_getaffinity(0)), 1)
    for b in (0, nblocks - 1):
        sh = oracle.encode_data(k, m, src[b * bs:(b + 1) * bs])
        assert all(np.array_equal(par[b, j], sh[k + j]) for j in range(m)), f"oracle self-check: parity of block {b}"
        assert all(dig[b, i].tobytes() == oracle.hh256(sh[i]) for i in range(k + m)), f"oracle self-check: digests of block {b}"
    return par, dig


def assert_blocks_equal(got, want, what, b0=0):
    """got / want: [blocks, rows, bytes]; names the first differing (block, row, byte) on failure."""
    if np.array_equal(got, want):
        return
    diff = got != want
    bad = np.nonzero(diff.reshape(diff.shape[0], -1).any(axis=1))[0]
    b = int(bad[0])
    row, byte = (int(v[0]) for v in np.nonzero(diff[b]))
    raise AssertionError(f"{what}: {bad.size} of {got.shape[0]} blocks differ; first: block {b0 + b}, row {row}, byte {byte} "
                         f"(got {got[b, row, byte]:#04x}, want {want[b, row, byte]:#04x})")


def device_random(nbytes, seed):
    import torch
    g = torch.Generator(device="cuda:0")
    g.manual_seed(seed)
    t = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
    for o in range(0, nbytes, 1 << 30):
        n = min(1 << 30, nbytes - o)
        t[o:o + n] = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda:0", generator=g)
    return t


def encode_and_check(mb, oracle, k, m, bs, nblocks, options, seed):
    """One mec_encode_blocks_device launch over `nblocks` blocks with the given codec options; every block's parity and digests
    against the oracle, the guard bytes of every parity row intact.  Returns (form counter deltas, last-launch record)."""
    import torch
    S = ceil_div(bs, k)
    n = k + m
    pitch = round_up(S, 16) + GUARD
    src = device_random(nblocks * bs, seed)
    par = torch.full((nblocks * m, pitch), FILL, dtype=torch.uint8, device="cuda:0")
    dig = torch.full((nblocks, n, 32), FILL, dtype=torch.uint8, device="cuda:0")
    c = mb.Codec(k, m, bs)
    try:
        for name, v in options.items():
            c.set_option(name, v)
        before = form_counts(c)
        c.encode_blocks_device(src.data_ptr(), nblocks * bs, par.data_ptr(), pitch, dig.data_ptr(),
                               torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        delta, last = form_delta(before, form_counts(c)), last_launch(c)
    finally:
        c.close()
    step = max(1, (256 * MiB) // bs)   # blocks come back (and go through the oracle) in slices: host memory stays flat at 1 MiB
    for b0 in range(0, nblocks, step):
        b1 = min(nblocks, b0 + step)
        want_par, want_dig = oracle_blocks(oracle, k, m, bs, src[b0 * bs:b1 * bs].cpu().numpy())
        assert_blocks_equal(dig[b0:b1].cpu().numpy(), want_dig, "digests", b0)
        got = par[b0 * m:b1 * m].view(b1 - b0, m, pitch).cpu().numpy()
        assert_blocks_equal(got[:, :, :S], want_par, "parity", b0)
        assert (got[:, :, S:] == FILL).all(), f"parity rows of blocks {b0}..{b1 - 1} were written past the shard end"
    return delta, last


# (k, m, S mod 16 of a 1 MiB block) of MEC_STATIC_CONFIGS (ec_engine.cu): the geometries with compile-time kernels
STATIC = [(12, 4, 6), (4, 2, 0), (16, 4, 0), (8, 8, 0), (8, 4, 0), (6, 2, 11), (2, 2, 0)]
DIRECT = [(k, m) for k, m, a in STATIC if a == 0]

# The 3-D fetch: tiles [0, tiles3d) of a shard arrive with one request per group of rows, the rest row by row.  (k, m, S, per-row
# fallback tiles at the end of the shard).  RS(12,4) needs two fallback tiles when S mod 256 < 86, RS(6,2) when < 75, the
# direct-fetch geometries (S mod 16 == 0) when 0 < S mod 256 < 32: each is tested on both sides of its edge.  The direct ones
# also run a full last tile (S mod 256 == 0) and partial ones.
FAST3D = [(12, 4, 12 * TILE + 70, 2), (12, 4, 12 * TILE + 86, 1), (6, 2, 12 * TILE + 59, 2), (6, 2, 12 * TILE + 75, 1)] + \
         [(k, m, 12 * TILE + s, fb) for k, m in DIRECT for s, fb in ((0, 1), (16, 2), (32, 1))]
# S mod 16 outside {0, sm16} for which a 16-byte multiple block size exists (k * S mod 16 < k), per k; odd or 2 mod 8 where one
# exists, so that the last 8-byte column of a row is partial
RUNTIME_S16 = {12: 2, 4: 4, 16: 5, 8: 2, 6: 3, 2: 8}


def multipass_options():
    return dict(eb=4, grid_mult=1)


def multipass_blocks(num_sms):
    return 8 * num_sms + 5   # 2 * num_sms + 2 groups of four on num_sms CTAs: two or three passes, a last group of one block


@pytest.mark.parametrize("k,m,S,fallback", [pytest.param(*c, id=f"rs{c[0]}_{c[1]}-S{c[2]}-fb{c[3]}") for c in FAST3D])
def test_static_fast3d(mb, oracle, num_sms, k, m, S, fallback):
    nblocks = multipass_blocks(num_sms)
    delta, last = encode_and_check(mb, oracle, k, m, bs_for(k, S), nblocks, multipass_options(), seed=S * 100 + k)
    assert delta == {"fast3d": 1}, delta
    assert last["num_sms"] == num_sms
    assert (last["last_eb"], last["last_grid"], last["last_tma_mode"], last["last_rows3d"], last["last_direct"]) == \
           (4, num_sms, TMA_BLOCKS2D, 1, int(S % 16 == 0)), last
    assert ceil_div(S, TILE) - last["last_tiles3d"] == fallback, last
    assert ceil_div(nblocks, last["last_eb"]) > last["last_grid"]


# (k, m, block size, options beyond eb = 4 / grid_mult = 1, form, direct fetch, TMA mode)
OTHER = [(12, 4, bs_for(12, 12 * TILE + 48), {}, "aligned", 1, TMA_BLOCKS2D),           # S % 16 == 0 differs from sm16
         (6, 2, bs_for(6, 12 * TILE + 48), {}, "aligned", 1, TMA_BLOCKS2D)]
OTHER += [c for k, m, a in STATIC for c in (
    (k, m, bs_for(k, 12 * TILE + RUNTIME_S16[k]), {}, "runtime", 0, TMA_BLOCKS2D),              # S % 16 in neither {0, sm16}
    (k, m, bs_for(k, 12 * TILE + (a or 16)), {"no_rows3d": 1}, "fast", int(a == 0), TMA_BLOCKS2D),  # 2-D boxes, one per row
    (k, m, bs_unaligned(k, 12 * TILE + RUNTIME_S16[k]), {}, "bytewise", 0, TMA_BYTEWISE))]     # block size not a multiple of 16


@pytest.mark.parametrize("k,m,bs,opts,form,direct,tma", [pytest.param(*c, id=f"rs{c[0]}_{c[1]}-{c[4]}-bs{c[2]}") for c in OTHER])
def test_static_other_forms(mb, oracle, num_sms, k, m, bs, opts, form, direct, tma):
    nblocks = multipass_blocks(num_sms)
    delta, last = encode_and_check(mb, oracle, k, m, bs, nblocks, dict(multipass_options(), **opts), seed=bs + k)
    assert delta == {form: 1}, delta
    assert (last["last_eb"], last["last_grid"], last["last_tma_mode"], last["last_rows3d"], last["last_direct"],
            last["last_tiles3d"]) == (4, num_sms, tma, 0, direct, 0), last
    assert ceil_div(nblocks, last["last_eb"]) > last["last_grid"]


# Default options at 1 MiB blocks: what a large device-resident encode runs.  (k, m, blocks as a function of the SM count, form,
# erasure blocks per CTA)
DEFAULT_1MIB = [
    # the misaligned 3-D encode's grid is capped at the raw-tile bytes in flight of five RS(12,4) CTAs per SM: some CTAs make a
    # second pass, and the last group holds three blocks
    pytest.param(12, 4, lambda s: 4 * 5 * s + 31, "fast3d", 4, id="rs12_4-fast3d-capped-grid"),
    # 661-1052 blocks: the CTA shrinks to two blocks so that there are two CTAs per SM, and the static runtime-alignment kernel runs
    pytest.param(12, 4, lambda s: 5 * s + 100, "runtime", 2, id="rs12_4-runtime-eb2"),
    pytest.param(6, 2, lambda s: 8 * s + 1, "fast3d", 4, id="rs6_2-fast3d"),
    pytest.param(8, 8, lambda s: 8 * s + 1, "fast3d", 4, id="rs8_8-fast3d-direct"),
]


@pytest.mark.parametrize("k,m,blocks,form,eb", DEFAULT_1MIB)
def test_default_options_1mib(mb, oracle, num_sms, k, m, blocks, form, eb):
    nblocks = blocks(num_sms)
    S = ceil_div(MiB, k)
    delta, last = encode_and_check(mb, oracle, k, m, MiB, nblocks, {}, seed=nblocks + k)
    assert delta == {form: 1}, delta
    assert last["last_eb"] == eb and last["last_rows3d"] == int(form == "fast3d"), last
    assert last["last_direct"] == int(S % 16 == 0 and eb == 4), last
    if form == "fast3d":
        assert ceil_div(S, TILE) - last["last_tiles3d"] == 1, last
    if k == 12 and form == "fast3d":
        assert last["last_grid"] == 5 * num_sms and ceil_div(nblocks, eb) > last["last_grid"], last


@pytest.mark.parametrize("static_groups", [0, 1], ids=["claimed", "static"])
@pytest.mark.parametrize("balance_grid", [0, 1], ids=["full_grid", "balanced_grid"])
def test_group_dealing(mb, oracle, num_sms, static_groups, balance_grid):
    """Groups of blocks dealt to CTAs statically or through the claim counter, on the full grid or one balanced so that every CTA
    makes the same number of passes: every block is encoded exactly once and right."""
    k, m, S = 12, 4, 12 * TILE + 70
    nblocks = multipass_blocks(num_sms)
    opts = dict(multipass_options(), static_groups=static_groups, balance_grid=balance_grid)
    delta, last = encode_and_check(mb, oracle, k, m, bs_for(k, S), nblocks, opts, seed=7000 + 2 * static_groups + balance_grid)
    assert delta == {"fast3d": 1}, delta
    ngroups = ceil_div(nblocks, 4)
    grid = num_sms if not balance_grid else ceil_div(ngroups, ceil_div(ngroups, num_sms))
    assert last["last_grid"] == grid and ngroups > grid, last


# Runtime-matrix encode (force_dynamic): one geometry per row chunk, rows fetched straight (S % 16 == 0) or re-aligned.
@pytest.mark.parametrize("k,m", [(8, 1), (10, 2), (12, 4)], ids=["rs8_1", "rs10_2", "rs12_4"])
@pytest.mark.parametrize("S,form", [(12 * TILE + 48, "dyn_aligned"), (12 * TILE + 2, "dyn_runtime")], ids=["aligned", "misaligned"])
def test_runtime_matrix_encode(mb, oracle, num_sms, k, m, S, form):
    nblocks = multipass_blocks(num_sms)
    opts = dict(multipass_options(), force_dynamic=1, jit=0)
    delta, last = encode_and_check(mb, oracle, k, m, bs_for(k, S), nblocks, opts, seed=S + 31 * k)
    assert delta == {form: 1}, delta
    assert (last["last_eb"], last["last_grid"], last["last_row_chunk"], last["last_rows3d"], last["last_direct"]) == \
           (4, num_sms, ROW_CHUNK[m], 0, int(form == "dyn_aligned")), last
    assert ceil_div(nblocks, 4) > last["last_grid"]


def test_nvrtc_encode_3d_fetch(mb, oracle, num_sms, jit_cache):
    """RS(10,4) has no compiled kernel: with jit = 1 the encode runs the NVRTC specialisation with the 3-D fetch (S mod 16 = 5,
    two fallback tiles), over several passes per CTA."""
    k, m, S = 10, 4, 16 * TILE + 5
    nblocks = multipass_blocks(num_sms)
    delta, last = encode_and_check(mb, oracle, k, m, bs_for(k, S), nblocks, dict(multipass_options(), jit=1), seed=1004)
    assert delta == {"jit": 1}, delta
    assert (last["last_eb"], last["last_grid"], last["last_rows3d"], last["last_direct"], last["last_row_chunk"]) == \
           (4, num_sms, 1, 0, -1), last
    assert ceil_div(S, TILE) - last["last_tiles3d"] == 2, last
    assert ceil_div(nblocks, 4) > last["last_grid"]


# ---------------------------------------------------------------- mec_reconstruct_device
RK, RM, RS = 12, 4, 12 * TILE + 70   # S mod 8 != 0: the last 8-byte column of every rebuilt row is a partial store


@pytest.fixture(scope="module")
def recon_truth(oracle, num_sms):
    """Shards and digests of every block of an RS(12,4) object from the oracle, as bitrot frames [n, nblocks, frame pitch]."""
    nblocks = multipass_blocks(num_sms)
    bs = bs_for(RK, RS)
    src = np.random.default_rng(4242).integers(0, 256, nblocks * bs, dtype=np.uint8)
    par, dig = oracle_blocks(oracle, RK, RM, bs, src)
    data = np.zeros((nblocks, RK * RS), dtype=np.uint8)
    data[:, :bs] = src.reshape(nblocks, bs)
    shards = np.concatenate([data.reshape(nblocks, RK, RS), par], axis=1)   # [nblocks, n, S]
    fp = round_up(32 + RS, 16)
    frames = np.zeros((RK + RM, nblocks, fp), dtype=np.uint8)
    frames[:, :, :32] = dig.transpose(1, 0, 2)
    frames[:, :, 32:32 + RS] = shards.transpose(1, 0, 2)
    return dict(nblocks=nblocks, shards=shards, dig=dig, frames=frames, fp=fp)


@pytest.mark.parametrize("layout,tma", [("separate", TMA_PER_INPUT), ("arena", TMA_RUNS)], ids=["separate", "arena"])
@pytest.mark.parametrize("erased", [(3,), (0, 13), (1, 5, 12, 15)], ids=["r1", "r2", "r4"])
@pytest.mark.parametrize("jit", [0, 1], ids=["jit0", "jit1"])
@pytest.mark.parametrize("flags", [0, 2], ids=["flags0", "flags2"])
def test_reconstruct_device(mb, num_sms, recon_truth, jit_cache, layout, tma, erased, jit, flags):
    """Rebuild r erased shards of every block from frames laid out in one arena (survivors at uniform strides: one 3-D tensor
    map per run) or at descending addresses (no two survivors at a uniform stride, as separately allocated frames are: one tensor
    map per survivor).  flags 2 = no digests for the rebuilt shards.  Then a flipped bit in a block that a CTA reaches on its second
    pass is flagged for exactly that block and reader."""
    import torch
    T = recon_truth
    nblocks, fp, n, S, r = T["nblocks"], T["fp"], RK + RM, RS, len(erased)
    frames_h = T["frames"] if layout == "arena" else T["frames"][::-1]
    store = torch.from_numpy(np.ascontiguousarray(frames_h)).to("cuda:0")
    frame = (lambda i: store[i]) if layout == "arena" else (lambda i: store[n - 1 - i])
    ptrs = [0 if i in erased else frame(i).data_ptr() for i in range(n)]
    readers = [i for i in range(n) if i not in erased][:RK]
    pitch = round_up(S, 16) + GUARD
    out = torch.full((nblocks * r, pitch), FILL, dtype=torch.uint8, device="cuda:0")
    dig = torch.full((nblocks, RK + r, 32), FILL, dtype=torch.uint8, device="cuda:0")
    cor = torch.zeros((nblocks, RK), dtype=torch.uint8, device="cuda:0")
    want = [int(i in erased) for i in range(n)]
    st = torch.cuda.current_stream().cuda_stream
    c = mb.Codec(RK, RM, bs_for(RK, RS))
    try:
        for name, v in dict(multipass_options(), jit=jit).items():
            c.set_option(name, v)
        before = form_counts(c)
        c.reconstruct_device(ptrs, fp, nblocks, want, flags, out.data_ptr(), pitch, dig.data_ptr(), cor.data_ptr(), st)
        torch.cuda.synchronize()
        delta, last = form_delta(before, form_counts(c)), last_launch(c)
        form = "jit" if jit else "dyn_aligned"
        assert delta == {form: 1}, delta
        assert (last["last_eb"], last["last_grid"], last["last_tma_mode"], last["last_direct"], last["last_row_chunk"]) == \
               (4, num_sms, tma, 1, -1 if jit else ROW_CHUNK[r]), last
        ngroups = ceil_div(nblocks, 4)
        assert ngroups > last["last_grid"]

        assert int(cor.sum().item()) == 0, "a clean frame was flagged"
        got = out.view(nblocks, r, pitch).cpu().numpy()
        assert_blocks_equal(got[:, :, :S], T["shards"][:, list(erased)], "rebuilt shards")
        assert (got[:, :, S:] == FILL).all(), "rebuilt rows were written past the shard end"
        hd = dig.cpu().numpy()
        assert_blocks_equal(hd[:, :RK], T["dig"][:, readers], "reader digests")
        if flags & 2:
            assert (hd[:, RK:] == FILL).all(), "digests of the rebuilt shards were written although not asked for"
        else:
            assert_blocks_equal(hd[:, RK:], T["dig"][:, list(erased)], "rebuilt-shard digests")

        # block 4 * grid + 6: group grid + 1, the second group CTA 1 takes
        b, pos = 4 * last["last_grid"] + 6, 5
        assert b // 4 >= last["last_grid"] and b < nblocks
        frame(readers[pos])[b, 32 + 1234] ^= 0x10
        c.reconstruct_device(ptrs, fp, nblocks, want, flags, out.data_ptr(), pitch, dig.data_ptr(), cor.data_ptr(), st)
        torch.cuda.synchronize()
        flagged = torch.nonzero(cor).cpu().tolist()
        assert flagged == [[b, pos]], flagged
    finally:
        c.close()
