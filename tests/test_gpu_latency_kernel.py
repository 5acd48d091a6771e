"""The latency kernel (small_rs_hh_kernel, ec_small.cuh) at the shard shapes and launch sizes that reach it, every erasure block
against the CPU oracle.

Every launch of at most 5 blocks per SM runs this kernel instead of the throughput kernel: small PutObjects, degraded GETs and
heals of that size, and every batch of the cross-request coalescer.  It has thirteen instantiations: one per compile-time
geometry (MEC_STATIC_CONFIGS, ec_engine.cu) and six runtime-matrix ones, by GF warps (3 when the launch's k + r <= 16, else 4)
and rows per pass of the matrix (1, 2 or 4).  Each test asserts from the dispatch counters that exactly one latency launch ran,
with one CTA per block and the intended row chunk, then compares the parity (or rebuilt shards) and the digests of every block
with the oracle.  Output rows are written at a pitch wider than the shard and pre-filled, so a store past the end of a shard
shows up in the guard bytes; the object sits in a buffer whose bytes behind it are pre-filled too, so a read past its end gives
wrong parity.

Shard lengths sit at the edges of the kernel's pipeline: a stage ("super-tile") is 256 bytes of every shard per GF warp, fetched
with cp.async three stages deep and handed to the hash warps over two buffers.  Block sizes are odd, so that the 16 blocks of
an object start each of their rows at all 16 offsets from a 16-byte boundary.
"""
import numpy as np
import pytest

from test_gpu_kernel_forms import (FILL, GUARD, assert_blocks_equal, bs_for, ceil_div, device_random, form_counts, form_delta,
                                   jit_cache, last_launch, mb, num_sms, oracle_blocks, round_up)

pytestmark = pytest.mark.gpu
MiB = 1 << 20
NFULL = 16           # full blocks of an object: row t of block b starts (b * bs + t * S) mod 16 bytes past a 16-byte boundary
DISPATCH_ENV = ("MEC_SMALL_BLOCKS", "MEC_EB", "MEC_FORCE_BYTEWISE", "MEC_FORCE_DYNAMIC", "MEC_JIT")
STATIC = {(12, 4), (4, 2), (16, 4), (8, 8), (8, 4), (6, 2), (2, 2)}   # MEC_STATIC_CONFIGS (ec_engine.cu)
ROW_CHUNK = {None: -1, 1: 0, 2: 1, 4: 2}                              # rows per pass -> last_row_chunk; None = compile-time matrix


@pytest.fixture(autouse=True)
def no_dispatch_env(monkeypatch):
    """Codec reads these when it is created: none of them may steer a launch here."""
    for name in DISPATCH_ENV:
        monkeypatch.delenv(name, raising=False)


def super_tile(gw):
    return 256 * gw


def latency_kernel(k, r, static):
    """(GF warps, rows per pass of the runtime matrix or None) of the latency kernel a launch of k inputs and r outputs runs."""
    return 3 if k + r <= 16 else 4, None if static else (1 if r <= 1 else (2 if r == 2 else 4))


def encode_kernel(k, m, opts):
    return latency_kernel(k, m, (k, m) in STATIC and not opts.get("force_dynamic"))


def encode_id(k, m, opts):
    gw, rc = encode_kernel(k, m, opts)
    return f"rs{k}_{m}{'-dyn' if opts.get('force_dynamic') else ''}-gw{gw}-{'static' if rc is None else f'rc{rc}'}"


def odd_bs(k, S):
    """The largest odd block size whose shards are S bytes: ceil(bs / k) == S."""
    bs = k * S if (k * S) % 2 else k * S - 1
    assert bs > 0 and ceil_div(bs, k) == S
    return bs


def oracle_block(oracle, k, m, data):
    """Parity [m, S] and digests [k + m, 32] of one erasure block: the oracle's Split + Encode and HighwayHash of every shard."""
    sh = oracle.encode_data(k, m, data)
    dig = np.stack([np.frombuffer(oracle.hh256(s, fast=True), dtype=np.uint8) for s in sh])
    return np.array(sh[k:], dtype=np.uint8).reshape(m, sh[0].size), dig


def assert_small_launch(run, grid, row_chunk, launches=1):
    assert run["launches"] == launches and run["delta"] == {"small": launches}, run
    last = run["last"]
    assert (last["last_eb"], last["last_grid"], last["last_tma_mode"], last["last_row_chunk"]) == (1, grid, -1, row_chunk), last


def encode(mb, k, m, bs, length, opts=None, digests=True, seed=0):
    """One mec_encode_blocks_device call over an object of `length` bytes, at a 16-byte boundary and followed by FILL bytes.
    m == 0 passes a NULL parity pointer, digests=False a NULL digest pointer.  -> (launch record, object, parity
    [blocks, m, pitch], digests [blocks, k + m, 32] or None), all on the host."""
    import torch
    S, nb = ceil_div(bs, k), ceil_div(length, bs)
    pitch = round_up(S, 16) + GUARD
    buf = torch.full((length + bs + 64,), FILL, dtype=torch.uint8, device="cuda:0")
    buf[:length] = device_random(length, seed)
    par = torch.full((nb, max(m, 1), pitch), FILL, dtype=torch.uint8, device="cuda:0")
    dig = torch.full((nb, k + m, 32), FILL, dtype=torch.uint8, device="cuda:0")
    c = mb.Codec(k, m, bs)
    try:
        for name, v in (opts or {}).items():
            c.set_option(name, v)
        before, launches = form_counts(c), c.launches
        c.encode_blocks_device(buf.data_ptr(), length, par.data_ptr() if m else 0, pitch, dig.data_ptr() if digests else 0,
                               torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        run = dict(delta=form_delta(before, form_counts(c)), launches=c.launches - launches, last=last_launch(c))
    finally:
        c.close()
    assert (buf[length:] == FILL).all(), "the object's neighbourhood was written"
    return run, buf[:length].cpu().numpy(), par[:, :m].cpu().numpy(), dig.cpu().numpy() if digests else None


def check_encode(oracle, k, m, bs, src, par, dig):
    """Parity and digests of every block of `src` (its last block may be short) against the oracle; each parity row keeps FILL
    from its block's shard length on."""
    S = ceil_div(bs, k)
    nfull, tail = divmod(src.size, bs)
    if (k - 1) * S < bs:
        want_par, want_dig = oracle_blocks(oracle, k, m, bs, src[:nfull * bs])
    else:   # S == 1 and k even: the last data shard is all padding
        per = [oracle_block(oracle, k, m, src[b * bs:(b + 1) * bs]) for b in range(nfull)]
        want_par, want_dig = np.stack([p for p, _ in per]), np.stack([d for _, d in per])
    assert_blocks_equal(par[:nfull, :, :S], want_par, "parity")
    assert (par[:nfull, :, S:] == FILL).all(), "parity rows were written past the shard end"
    if dig is not None:
        assert_blocks_equal(dig[:nfull], want_dig, "digests")
    if tail:
        St = ceil_div(tail, k)
        tp, td = oracle_block(oracle, k, m, src[nfull * bs:])
        assert_blocks_equal(par[nfull:, :, :St], tp[None], "tail-block parity", nfull)
        assert (par[nfull, :, St:] == FILL).all(), f"tail-block parity rows were written past its {St}-byte shards"
        if dig is not None:
            assert_blocks_equal(dig[nfull:], td[None], "tail-block digests", nfull)


# ---------------------------------------------------------------- mec_encode_blocks_device: every instantiation
# (k, m, options): geometries without a compiled kernel (and force_dynamic) run the runtime-matrix kernel with the encode matrix
GEOMETRIES = [(12, 4, {}), (4, 2, {}), (8, 8, {}), (8, 4, {}), (6, 2, {}), (2, 2, {}),      # compile-time, 3 GF warps
              (16, 4, {}),                                                                 # compile-time, 4 GF warps
              (9, 1, {}), (3, 0, {}),                                                      # runtime, GW 3, RC 1 (r = 0: hash only)
              (10, 2, {}),                                                                 # runtime, GW 3, RC 2
              (10, 4, {}), (5, 3, {}), (7, 5, {}), (12, 4, {"force_dynamic": 1}),         # RC 4: padded chunk, two passes
              (17, 1, {}), (17, 0, {}), (15, 2, {}),                                       # runtime, GW 4, RC 1 / 2
              (20, 4, {}), (32, 16, {})]                                                   # RC 4: four passes, 3 hash warps
# one kernel per compile-time geometry, one per (GF warps, row chunk) of the runtime matrix
assert len({("static", k, m) if encode_kernel(k, m, o)[1] is None else ("runtime",) + encode_kernel(k, m, o)
            for k, m, o in GEOMETRIES}) == 13


def encode_row_chunk(k, m, opts):
    return ROW_CHUNK[encode_kernel(k, m, opts)[1]]


def encode_super(k, m):
    return super_tile(encode_kernel(k, m, {})[0])


def shard_lengths(k, m):
    sup = encode_super(k, m)
    # partial 8-byte columns, one packet +- 1, one stage +- 1, a partial third stage, seven stages (both rings wrap more than
    # once), and the shard of a 1 MiB block
    return [1, 5, 8, 13, 31, 32, 33, sup - 1, sup, sup + 1, 2 * sup + 7, 6 * sup + 29, ceil_div(MiB, k)]


SWEEP = [pytest.param(k, m, o, S, id=f"{encode_id(k, m, o)}-S{S}") for k, m, o in GEOMETRIES for S in shard_lengths(k, m)]


@pytest.mark.parametrize("k,m,opts,S", SWEEP)
def test_encode_shard_lengths(mb, oracle, k, m, opts, S):
    """16 odd-sized blocks and a short one in one launch (a 1 MiB block alone for the last S): every row at every lead."""
    if S == ceil_div(MiB, k):
        bs, length = MiB, MiB
    else:
        bs = odd_bs(k, S)
        length = NFULL * bs + ((bs // 3) | 1 if bs > 1 else 0)
    run, src, par, dig = encode(mb, k, m, bs, length, opts, seed=S * 64 + k)
    assert_small_launch(run, ceil_div(length, bs), encode_row_chunk(k, m, opts))
    check_encode(oracle, k, m, bs, src, par, dig)


@pytest.mark.parametrize("k,m,S", [(12, 4, 2 * 768 + 7), (16, 4, 2 * 1024 + 7)], ids=["rs12_4-gw3", "rs16_4-gw4"])
def test_encode_aligned_blocks(mb, oracle, k, m, S):
    """Block size a multiple of 16: every block starts on a 16-byte boundary."""
    bs = bs_for(k, S)
    run, src, par, dig = encode(mb, k, m, bs, NFULL * bs, seed=S + k)
    assert_small_launch(run, NFULL, -1)
    check_encode(oracle, k, m, bs, src, par, dig)


def tail_bs(k, m):
    return odd_bs(k, 2 * encode_super(k, m) + 7)


def tail_lengths(k, m):
    sup = encode_super(k, m)
    # one byte (rows 1..k-1 all padding), about one byte per row, shards of one stage -+ 1, one byte short of a full block
    return sorted({1, k - 1, k, k + 1, k * (sup - 1) - k // 2, k * (sup + 1) - k // 2, tail_bs(k, m) - 1})


TAILS = [pytest.param(k, m, o, t, id=f"{encode_id(k, m, o)}-tail{t}") for k, m, o in GEOMETRIES for t in tail_lengths(k, m)]


@pytest.mark.parametrize("k,m,opts,tail", TAILS)
def test_encode_tail_block(mb, oracle, k, m, opts, tail):
    """The object's short last block rides in the same launch with its own shard length (tail_block / tail_in_off)."""
    bs = tail_bs(k, m)
    assert 0 < tail < bs
    run, src, par, dig = encode(mb, k, m, bs, NFULL * bs + tail, opts, seed=tail * 8 + k)
    assert_small_launch(run, NFULL + 1, encode_row_chunk(k, m, opts))
    check_encode(oracle, k, m, bs, src, par, dig)


@pytest.mark.parametrize("k,m", [(12, 4), (10, 4)], ids=["rs12_4-static", "rs10_4-rc4"])
def test_encode_parity_only(mb, oracle, k, m):
    """d_digests == NULL: nothing is hashed, the parity is still exact."""
    bs = odd_bs(k, 768 + 1)
    run, src, par, _ = encode(mb, k, m, bs, NFULL * bs + 5 * k + 3, digests=False, seed=k + m)
    assert_small_launch(run, NFULL + 1, encode_row_chunk(k, m, {}))
    check_encode(oracle, k, m, bs, src, par, None)


# ---------------------------------------------------------------- mec_reconstruct_device
DATA_ONLY, NO_OUTPUT_DIGESTS = 1, 2   # MEC_RECONSTRUCT_* flags
RECON_BLOCKS = 17
# (id, k, m, unavailable shards, wanted shards, data only)
RECON = [("rs12_4-r0", 12, 4, (2,), (), False),   # nothing to rebuild: hash and verify the readers only
         ("rs12_4-r1", 12, 4, (3,), (3,), False),
         ("rs12_4-r2", 12, 4, (0, 13), (0, 13), False),
         ("rs12_4-r3", 12, 4, (1, 7, 14), (1, 7, 14), False),
         ("rs12_4-r4", 12, 4, (1, 5, 12, 15), (1, 5, 12, 15), False),
         ("rs16_4-r1", 16, 4, (5,), (5,), False),   # k + r > 16: four GF warps for one rebuilt shard
         ("rs16_4-r2", 16, 4, (0, 17), (0, 17), False),
         ("rs16_4-r4", 16, 4, (2, 9, 16, 19), (2, 9, 16, 19), False),
         ("rs8_8-r8", 8, 8, (0, 2, 4, 6, 9, 11, 13, 15), (0, 2, 4, 6, 9, 11, 13, 15), False),
         ("rs8_8-data_only-r3", 8, 8, (1, 3, 6, 8, 9, 10, 12, 14), (1, 3, 6, 8, 9, 10, 12, 14), True),
         # the widest launch: 7 warps and 219,712 bytes of shared memory
         ("rs32_16-r16", 32, 16, tuple(range(1, 48, 3)), tuple(range(1, 48, 3)), False)]


def recon_plan(k, m, unavailable, wanted, data_only):
    """(readers, rebuilt shards) of mec_reconstruct_device: the first k available shards are read."""
    readers = [i for i in range(k + m) if i not in unavailable][:k]
    return readers, [i for i in sorted(wanted) if i not in readers and not (data_only and i >= k)]


def recon_lengths(k, m, unavailable, wanted, data_only):
    sup = super_tile(latency_kernel(k, len(recon_plan(k, m, unavailable, wanted, data_only)[1]), False)[0])
    return [13, sup - 1, sup + 1, 6 * sup + 29]


RECON_CASES = [pytest.param(*case, S, flags, id=f"{name}-S{S}-flags{flags}")
               for name, *case in RECON for S in recon_lengths(*case) for flags in (0, NO_OUTPUT_DIGESTS)]


@pytest.mark.parametrize("k,m,unavailable,wanted,data_only,S,flags", RECON_CASES)
def test_reconstruct(mb, oracle, k, m, unavailable, wanted, data_only, S, flags):
    """Rebuild the wanted shards of every block from the first k available frames, each shard's frames in an arena of its own
    that starts (7 * shard) mod 16 bytes past a 16-byte boundary.  Then a bit flipped in a reader's first shard byte, its last
    shard byte (in the hash's remainder packet) or either half of its stored digest, in the first or the last block, flags
    exactly that block and reader."""
    import torch
    n, nb = k + m, RECON_BLOCKS
    readers, targets = recon_plan(k, m, unavailable, wanted, data_only)
    r = len(targets)
    src = np.random.default_rng(S * 100 + n + r).integers(0, 256, nb * k * S, dtype=np.uint8)
    par, dig = oracle_blocks(oracle, k, m, k * S, src)
    shards = np.concatenate([src.reshape(nb, k, S), par], axis=1)      # [nb, n, S]
    fp = round_up(32 + S, 16)
    frames = {}
    for i in range(n):
        if i in unavailable:
            continue
        lead = 7 * i % 16
        h = np.full(lead + nb * fp, FILL, dtype=np.uint8)
        f = h[lead:].reshape(nb, fp)
        f[:, :32], f[:, 32:32 + S] = dig[:, i], shards[:, i]
        frames[i] = torch.from_numpy(h).to("cuda:0")[lead:].view(nb, fp)
    ptrs = [frames[i].data_ptr() if i in frames else 0 for i in range(n)]
    want = [int(i in wanted) for i in range(n)]
    flags |= DATA_ONLY if data_only else 0
    pitch = round_up(S, 16) + GUARD
    out = torch.full((nb, max(r, 1), pitch), FILL, dtype=torch.uint8, device="cuda:0")
    dg = torch.full((nb, k + r, 32), FILL, dtype=torch.uint8, device="cuda:0")
    cor = torch.zeros((nb, k), dtype=torch.uint8, device="cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    c = mb.Codec(k, m, k * S)
    try:
        def reconstruct():
            before, launches = form_counts(c), c.launches
            c.reconstruct_device(ptrs, fp, nb, want, flags, out.data_ptr() if r else 0, pitch, dg.data_ptr(), cor.data_ptr(), st)
            torch.cuda.synchronize()
            assert_small_launch(dict(delta=form_delta(before, form_counts(c)), launches=c.launches - launches, last=last_launch(c)),
                                nb, ROW_CHUNK[latency_kernel(k, r, False)[1]])

        reconstruct()
        assert int(cor.sum().item()) == 0, "a clean frame was flagged"
        got = out[:, :r].cpu().numpy()
        assert_blocks_equal(got[:, :, :S], shards[:, targets], "rebuilt shards")
        assert (got[:, :, S:] == FILL).all(), "rebuilt rows were written past the shard end"
        hd = dg.cpu().numpy()
        assert_blocks_equal(hd[:, :k], dig[:, readers], "reader digests")
        if flags & NO_OUTPUT_DIGESTS:
            assert (hd[:, k:] == FILL).all(), "digests of the rebuilt shards were written although not asked for"
        else:
            assert_blocks_equal(hd[:, k:], dig[:, targets], "rebuilt-shard digests")

        for b, pos in ((0, k - 1), (nb - 1, 0)):
            f = frames[readers[pos]]
            for byte, bit in ((32, 0x01), (32 + S - 1, 0x80), (5, 0x04), (29, 0x20)):   # digest bytes 0-15 / 16-31: two lanes
                f[b, byte] ^= bit
                cor.zero_()
                reconstruct()
                f[b, byte] ^= bit
                flagged = torch.nonzero(cor).cpu().tolist()
                assert flagged == [[b, pos]], (b, byte, flagged)
    finally:
        c.close()


# ---------------------------------------------------------------- which launches take the latency kernel
DK, DM, DS = 12, 4, 13   # 155-byte blocks


@pytest.mark.parametrize("extra", [0, 1], ids=["limit", "limit_plus_1"])
def test_dispatch_small_limit(mb, oracle, num_sms, extra):
    """5 blocks per SM take the latency kernel; one more block takes a throughput form, with the same bytes."""
    bs = odd_bs(DK, DS)
    nb = 5 * num_sms + extra
    run, src, par, dig = encode(mb, DK, DM, bs, nb * bs, dict(jit=0), seed=nb)
    assert run["last"]["num_sms"] == num_sms
    if extra:
        assert run["launches"] == 1 and sum(run["delta"].values()) == 1 and "small" not in run["delta"], run
    else:
        assert_small_launch(run, nb, -1)
    check_encode(oracle, DK, DM, bs, src, par, dig)


@pytest.mark.parametrize("nb", [7, 8], ids=["N", "N_plus_1"])
def test_dispatch_small_blocks_option(mb, oracle, nb):
    """small_blocks = N: launches of at most N blocks take the latency kernel."""
    bs = odd_bs(DK, DS)
    run, src, par, dig = encode(mb, DK, DM, bs, nb * bs, dict(small_blocks=7, jit=0), seed=nb)
    if nb > 7:
        assert run["launches"] == 1 and sum(run["delta"].values()) == 1 and "small" not in run["delta"], run
    else:
        assert_small_launch(run, nb, -1)
    check_encode(oracle, DK, DM, bs, src, par, dig)


@pytest.mark.parametrize("opts", [dict(eb=1), dict(force_bytewise=1), dict(jit=1), dict(small_blocks=0)],
                         ids=["eb1", "force_bytewise", "jit1", "small_blocks0"])
def test_dispatch_options_avoid_small(mb, oracle, jit_cache, opts):
    """Each of these options keeps even a one-block launch on the throughput kernel."""
    bs = odd_bs(DK, DS)
    run, src, par, dig = encode(mb, DK, DM, bs, bs, opts, seed=len(str(opts)))
    assert run["launches"] == 1 and sum(run["delta"].values()) == 1 and "small" not in run["delta"], run
    check_encode(oracle, DK, DM, bs, src, par, dig)


def test_dispatch_tail_past_limit(mb, oracle, num_sms):
    """5 full blocks per SM and a short one: the full blocks fill a latency launch, the short one takes a second."""
    bs = odd_bs(DK, DS)
    nfull = 5 * num_sms
    run, src, par, dig = encode(mb, DK, DM, bs, nfull * bs + 7, seed=nfull)
    assert_small_launch(run, 1, -1, launches=2)
    check_encode(oracle, DK, DM, bs, src, par, dig)
