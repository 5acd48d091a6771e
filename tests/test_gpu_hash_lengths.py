"""HighwayHash-256 bitrot digests at every remainder length and tile position, on every kernel form that hashes, against the CPU
oracle.

Every streaming-bitrot frame starts with the HighwayHash-256 of its shard, and every read compares it: a form that hashes the
wrong bytes at some shard lengths makes healthy data read as corrupt (writer side) or lets corruption through (reader side).
The hash arithmetic is shared by all forms; what differs is where each form finds the bytes.  In the throughput kernel
(ec_kernel.cuh) the last packets of a shard sit in its last 256-byte tile, the remainder (S mod 32 bytes) at
(npk * 32) mod 256 with npk = S / 32, and with the direct TMA fetch (rows 16-byte aligned) that tile is in one of two buffers
chosen by the parity of a tile counter that runs on across the groups of blocks a CTA takes.  The latency kernel (ec_small.cuh)
finds them in 768- or 1024-byte stages.

Shard lengths S = 256 * T + x: x = 33 * j mod 256 for j = 0..31 gives every S mod 32 once and every packet position of the last
tile ((S mod 256) / 32) four times; x = 1, 31, 32, 224, 255 are the edges.  T = 0 is one partial tile (S < 32: no whole
packet), T = 12 and 13 give 13 / 14 tiles (12 / 13 for x = 0): the direct fetch's second group of a CTA starts in either buffer.
The forms that take only some residues of S mod 16 run their own classes across the 8 packet positions.  Every test asserts from
the "form_*" / "last_*" dispatch counters which form ran, so a dispatch change cannot quietly skip a case.
"""
import numpy as np
import pytest

import selftest_goldens as G
import test_gpu_kernel_forms as kernel_forms
from test_gpu_kernel_forms import (FILL, GUARD, ROW_CHUNK, STATIC, TMA_BLOCKS2D, TMA_BYTEWISE, TMA_PER_INPUT, TMA_RUNS,
                                   assert_blocks_equal, bs_for, bs_unaligned, ceil_div, encode_and_check, form_counts, form_delta,
                                   jit_cache, last_launch, mb, multipass_blocks, multipass_options, num_sms, oracle_blocks,
                                   round_up)

gpu = pytest.mark.gpu
TILE = 256
DISPATCH_ENV = ("MEC_SMALL_BLOCKS", "MEC_EB", "MEC_FORCE_BYTEWISE", "MEC_FORCE_DYNAMIC", "MEC_JIT")

TILES = (0, 12, 13)
X_RECIPE = sorted({33 * j % TILE for j in range(32)} | {1, 31, 32, 224, 255})
LENGTHS = [TILE * T + x for T in TILES for x in X_RECIPE if TILE * T + x > 0]   # S = 0 only in the empty-message tests


def class_lengths(c):
    """S mod 32 == c at every packet position of the last tile, for every T."""
    return [TILE * T + 32 * p + c for T in TILES for p in range(8) if TILE * T + 32 * p + c > 0]


ALIGNED16 = class_lengths(0) + class_lengths(16)        # the forms that fetch 16-byte aligned rows take only these
SWEEP_LENGTHS = sorted(set(LENGTHS) | set(ALIGNED16))


@pytest.fixture(autouse=True)
def no_dispatch_env(monkeypatch):
    """Codec reads these when it is created: none of them may steer a launch here."""
    for name in DISPATCH_ENV:
        monkeypatch.delenv(name, raising=False)


def test_length_recipe_covers_every_class():
    """The recipe reaches every remainder length and every packet position at every tile count, S < 32, and both parities of
    the tile count (the direct fetch's buffer of a CTA's second group); the aligned classes reach every packet position."""
    for T in TILES:
        xs = [S - TILE * T for S in LENGTHS if S // TILE == T]
        assert {x % 32 for x in xs} == set(range(32)), T
        assert {x // 32 for x in xs} == set(range(8)), T
    assert 0 not in LENGTHS and any(S < 32 for S in LENGTHS)
    for T in TILES[1:]:
        assert {ceil_div(S, TILE) % 2 for S in LENGTHS if S // TILE == T} == {0, 1}, T
    for c in (0, 16):
        for T in TILES:
            positions = {(S % TILE) // 32 for S in class_lengths(c) if S // TILE == T}
            assert positions == set(range(1 if (c, T) == (0, 0) else 0, 8)), (c, T)   # S = 0: not a shard


def has_bs16(k, S):
    """Is there a block size that is a multiple of 16 and has shards of S bytes (see bs_for)?"""
    return (k * S) % 16 < k


# ---------------------------------------------------------------- mec_hh256_batch: the hash-only forms
HH_FORMS = ("small", "dyn_bytewise", "dyn_aligned")
SMALL_COUNT = 5   # messages of a latency-kernel launch: one CTA each


def hh_setup(form, num_sms):
    """(options, message count) that make a hash-only launch take `form`: the latency kernel below its block limit, or the
    throughput kernel with four messages per CTA and one CTA per SM, so that CTAs take two or three groups and the last group
    holds one message."""
    if form == "small":
        return {}, SMALL_COUNT
    return dict(multipass_options(), **({"force_bytewise": 1} if form == "dyn_bytewise" else {})), multipass_blocks(num_sms)


def hh_batch(c, msgs, S, count):
    """One mec_hh256_batch call -> (digests [count, 32], form counter deltas, last-launch record, launches)."""
    before, launches = form_counts(c), c.launches
    got = c.hh256_batch(msgs, S, count)
    return got, form_delta(before, form_counts(c)), last_launch(c), c.launches - launches


def assert_hh_form(form, delta, last, count, num_sms):
    assert delta == {form: 1}, delta
    if form == "small":
        assert (last["last_eb"], last["last_grid"], last["last_tma_mode"]) == (1, count, -1), last
    else:
        tma, direct = (TMA_BYTEWISE, 0) if form == "dyn_bytewise" else (TMA_PER_INPUT, 1)
        assert (last["last_eb"], last["last_grid"], last["last_tma_mode"], last["last_direct"]) == (4, num_sms, tma, direct), last
        assert ceil_div(count, 4) > last["last_grid"], last


def oracle_hh(oracle, msgs, S):
    """HighwayHash-256 of each S-byte message of `msgs` [count, 32], from the oracle (k = 1, no parity: a block is a shard)."""
    return oracle_blocks(oracle, 1, 0, S, np.ascontiguousarray(msgs).reshape(-1))[1][:, 0]


@gpu
@pytest.mark.parametrize("form", HH_FORMS)
@pytest.mark.parametrize("S", LENGTHS, ids=[f"S{S}" for S in LENGTHS])
def test_hh_batch_lengths(mb, oracle, num_sms, form, S):
    opts, count = hh_setup(form, num_sms)
    msgs = np.random.default_rng(S * 8 + HH_FORMS.index(form)).integers(0, 256, (count, S), dtype=np.uint8)
    c = mb.Codec(2, 2)
    try:
        for name, v in opts.items():
            c.set_option(name, v)
        got, delta, last, _ = hh_batch(c, msgs, S, count)
    finally:
        c.close()
    assert_hh_form(form, delta, last, count, num_sms)
    assert_blocks_equal(got[:, None], oracle_hh(oracle, msgs, S)[:, None], f"{form} digests")


@gpu
@pytest.mark.parametrize("count", [1, 3, "over_limit"])
def test_hh_batch_empty_message(mb, oracle, num_sms, count):
    """msg_len == 0: nothing is staged or fetched, every digest is HH256 of the empty message (the reference's golden), also
    for more messages than a latency-kernel launch takes."""
    count = 5 * num_sms + 1 if count == "over_limit" else count
    want = bytes.fromhex(G.DERIVED_HH[0])
    assert oracle.hh256(b"") == want
    c = mb.Codec(2, 2)
    try:
        got, delta, last, launches = hh_batch(c, np.zeros(0, dtype=np.uint8), 0, count)
    finally:
        c.close()
    assert launches == 1 and delta == {"dyn_bytewise": 1}, delta
    assert last["last_tma_mode"] == TMA_BYTEWISE, last
    assert got.shape == (count, 32) and all(got[i].tobytes() == want for i in range(count))


@gpu
def test_hh_batch_no_messages_is_no_launch(mb):
    """count == 0: no digest, no kernel."""
    c = mb.Codec(2, 2)
    try:
        got, delta, _, launches = hh_batch(c, np.zeros(0, dtype=np.uint8), 100, 0)
    finally:
        c.close()
    assert got.shape == (0, 32) and launches == 0 and delta == {}, delta


STALE_LENGTHS = [1, 31, 33, 255, 12 * TILE + 99, 13 * TILE + 255]
STALE_LONG = 14 * TILE   # a multiple of 16: the 0xFF messages cover their staging rows without gaps


@gpu
@pytest.mark.parametrize("form", HH_FORMS)
def test_hh_batch_stale_staging(mb, oracle, num_sms, form):
    """Messages are staged in rows of round_up(S, 16) bytes of a buffer the codec keeps; only S bytes of each row are written.
    After a call with longer 0xFF messages the rest of every row still holds 0xFF: the digests must not see it."""
    opts, count = hh_setup(form, num_sms)
    c = mb.Codec(2, 2)
    try:
        for name, v in opts.items():
            c.set_option(name, v)
        ff = np.full((count, STALE_LONG), 0xFF, dtype=np.uint8)
        for S in STALE_LENGTHS:
            got, delta, last, _ = hh_batch(c, ff, STALE_LONG, count)
            assert_hh_form(form, delta, last, count, num_sms)
            assert got[0].tobytes() == oracle.hh256(ff[0]) and (got == got[0]).all(), "0xFF digests"
            msgs = np.random.default_rng(S).integers(0, 256, (count, S), dtype=np.uint8)
            got, delta, last, _ = hh_batch(c, msgs, S, count)
            assert_hh_form(form, delta, last, count, num_sms)
            assert_blocks_equal(got[:, None], oracle_hh(oracle, msgs, S)[:, None], f"{form} digests after 0xFF rows, S = {S}")
    finally:
        c.close()


# ---------------------------------------------------------------- mec_encode_blocks_device: digests of all k + m shards
def static_case(k, sm16, S):
    """(block size, form, direct fetch, TMA mode) of an encode of the compile-time geometry (k, m, sm16) with eb = 4: a block
    size that is a multiple of 16 where one exists, else the byte-wise loader.  Rows too short for a 3-D request (less than a
    tile) take the 2-D form of the sm16 kernel."""
    if not has_bs16(k, S):
        return bs_unaligned(k, S), "bytewise", 0, TMA_BYTEWISE
    if S % 16 == sm16:
        return bs_for(k, S), "fast" if S < TILE else "fast3d", int(sm16 == 0), TMA_BLOCKS2D
    return bs_for(k, S), "aligned" if S % 16 == 0 else "runtime", int(S % 16 == 0), TMA_BLOCKS2D


def check_encode_launch(delta, last, form, direct, tma, num_sms, nblocks):
    assert delta == {form: 1}, delta
    assert (last["last_eb"], last["last_grid"], last["last_tma_mode"], last["last_direct"], last["last_rows3d"]) == \
           (4, num_sms, tma, direct, int(form == "fast3d")), last
    assert ceil_div(nblocks, 4) > last["last_grid"]


SWEEP_STATIC = [(k, m, sm16, S) for k, m, sm16 in STATIC if (k, m) in ((12, 4), (6, 2)) for S in SWEEP_LENGTHS]


@gpu
@pytest.mark.parametrize("k,m,sm16,S", [pytest.param(*c, id=f"rs{c[0]}_{c[1]}-{static_case(c[0], c[2], c[3])[1]}-S{c[3]}")
                                        for c in SWEEP_STATIC])
def test_encode_static_lengths(mb, oracle, num_sms, k, m, sm16, S):
    bs, form, direct, tma = static_case(k, sm16, S)
    nblocks = multipass_blocks(num_sms)
    delta, last = encode_and_check(mb, oracle, k, m, bs, nblocks, multipass_options(), seed=S * 32 + k)
    check_encode_launch(delta, last, form, direct, tma, num_sms, nblocks)


# the compile-time kernels for S mod 16 == sm16: both residues of S mod 32 at every packet position
FAST = [(k, m, sm16, S) for k, m, sm16 in STATIC for c in (sm16, sm16 + 16) for S in class_lengths(c)]


def oracle_blocks_padded(oracle, k, m, bs, src):
    """oracle_blocks, also for blocks that leave more than the last data shard as padding ((k - 1) * S >= bs: RS(12,4) with
    64-byte blocks of 6-byte shards), which the oracle's block encoder does not take: those from the scalar Split + Encode and
    HighwayHash of every block."""
    S = ceil_div(bs, k)
    if (k - 1) * S < bs:
        return oracle_blocks(oracle, k, m, bs, src)
    nblocks = src.size // bs
    sh = [oracle.encode_data(k, m, src[b * bs:(b + 1) * bs]) for b in range(nblocks)]
    par = np.array([s[k:] for s in sh], dtype=np.uint8).reshape(nblocks, m, S)
    dig = np.array([[np.frombuffer(oracle.hh256(x), dtype=np.uint8) for x in s] for s in sh]).reshape(nblocks, k + m, 32)
    return par, dig


@gpu
@pytest.mark.parametrize("k,m,sm16,S", [pytest.param(*c, id=f"rs{c[0]}_{c[1]}-{static_case(c[0], c[2], c[3])[1]}-S{c[3]}")
                                        for c in FAST])
def test_encode_fast_classes(mb, oracle, num_sms, monkeypatch, k, m, sm16, S):
    bs, form, direct, tma = static_case(k, sm16, S)
    assert form in ("fast", "fast3d")
    monkeypatch.setattr(kernel_forms, "oracle_blocks", oracle_blocks_padded)   # encode_and_check's reference
    nblocks = multipass_blocks(num_sms)
    delta, last = encode_and_check(mb, oracle, k, m, bs, nblocks, multipass_options(), seed=S * 32 + k + 1)
    check_encode_launch(delta, last, form, direct, tma, num_sms, nblocks)


def dynamic_case(k, S):
    if not has_bs16(k, S):
        return bs_unaligned(k, S), "dyn_bytewise", 0, TMA_BYTEWISE
    return bs_for(k, S), "dyn_aligned" if S % 16 == 0 else "dyn_runtime", int(S % 16 == 0), TMA_BLOCKS2D


# runtime-matrix encode: one geometry per row chunk
SWEEP_DYNAMIC = [(k, m, S) for k, m in ((8, 1), (10, 2), (12, 4)) for S in SWEEP_LENGTHS]


@gpu
@pytest.mark.parametrize("k,m,S", [pytest.param(*c, id=f"rs{c[0]}_{c[1]}-{dynamic_case(c[0], c[2])[1]}-S{c[2]}")
                                   for c in SWEEP_DYNAMIC])
def test_encode_runtime_matrix_lengths(mb, oracle, num_sms, k, m, S):
    bs, form, direct, tma = dynamic_case(k, S)
    nblocks = multipass_blocks(num_sms)
    opts = dict(multipass_options(), force_dynamic=1, jit=0)
    delta, last = encode_and_check(mb, oracle, k, m, bs, nblocks, opts, seed=S * 32 + k + 2)
    check_encode_launch(delta, last, form, direct, tma, num_sms, nblocks)
    assert last["last_row_chunk"] == ROW_CHUNK[m], last


@gpu
@pytest.mark.parametrize("S", [12 * TILE + 231, 13 * TILE + 165], ids=["S3303", "S3493"])
def test_encode_nvrtc_lengths(mb, oracle, num_sms, jit_cache, S):
    """RS(10,4) has no compiled kernel: jit = 1 runs the NVRTC specialisation for S mod 16 (odd remainders at packet positions
    7 and 5 of the last tile)."""
    k, m = 10, 4
    nblocks = multipass_blocks(num_sms)
    delta, last = encode_and_check(mb, oracle, k, m, bs_for(k, S), nblocks, dict(multipass_options(), jit=1), seed=S + 10)
    assert delta == {"jit": 1}, delta
    assert (last["last_eb"], last["last_grid"], last["last_row_chunk"]) == (4, num_sms, -1), last
    assert ceil_div(nblocks, 4) > last["last_grid"]


# ---------------------------------------------------------------- mec_reconstruct_device: reader and output digests
RK, RM = 12, 4
ERASED = (1, 5, 12, 15)
READERS = [i for i in range(RK + RM) if i not in ERASED][:RK]
RECON_S = [2 * 32 + 2, 12 * TILE + 255, 13 * TILE + 99]   # S mod 32 = 2, 31, 3 at packet positions 2, 7, 3; 1, 13, 14 tiles
PAD = 64           # frame pitch = round_up(32 + S, 16) + PAD: the bytes from 32 + S on are random
SMALL_BLOCKS = 17  # blocks of a latency-kernel reconstruct
# (form, frame layout, options)
RECON_FORMS = [("dyn_aligned", "separate", dict(multipass_options(), jit=0)),
               ("dyn_aligned", "arena", dict(multipass_options(), jit=0)),
               ("dyn_bytewise", "arena", dict(multipass_options(), force_bytewise=1, jit=0)),
               ("small", "arena", {})]


@pytest.fixture(scope="module")
def recon_frames(oracle, num_sms):
    """S -> shards and digests of every block of an RS(12,4) object from the oracle, as bitrot frames [n, nblocks, pitch] whose
    bytes past the shard are random."""
    cache = {}

    def get(S):
        if S not in cache:
            nblocks = multipass_blocks(num_sms)
            bs = bs_for(RK, S)
            rng = np.random.default_rng(S)
            src = rng.integers(0, 256, nblocks * bs, dtype=np.uint8)
            par, dig = oracle_blocks(oracle, RK, RM, bs, src)
            data = np.zeros((nblocks, RK * S), dtype=np.uint8)
            data[:, :bs] = src.reshape(nblocks, bs)
            shards = np.concatenate([data.reshape(nblocks, RK, S), par], axis=1)   # [nblocks, n, S]
            fp = round_up(32 + S, 16) + PAD
            frames = rng.integers(0, 256, (RK + RM, nblocks, fp), dtype=np.uint8)
            frames[:, :, :32] = dig.transpose(1, 0, 2)
            frames[:, :, 32:32 + S] = shards.transpose(1, 0, 2)
            cache[S] = dict(nblocks=nblocks, bs=bs, shards=shards, dig=dig, frames=frames, fp=fp)
        return cache[S]

    return get


@gpu
@pytest.mark.parametrize("form,layout,opts", [pytest.param(*f, id=f"{f[0]}-{f[1]}") for f in RECON_FORMS])
@pytest.mark.parametrize("S", RECON_S, ids=[f"S{S}" for S in RECON_S])
def test_reconstruct_digests_ignore_frame_padding(mb, num_sms, recon_frames, form, layout, opts, S):
    """Rebuild four erased shards of every block from frames whose pitch padding is random: reader and rebuilt-shard digests and
    the rebuilt rows match the oracle.  A bit flipped in a reader's first remainder byte or last shard byte, in a block that a
    CTA takes on its second pass (the last block for the latency kernel), flags exactly that block and reader; a bit flipped in
    the padding flags nothing."""
    import torch
    T = recon_frames(S)
    fp, n, r = T["fp"], RK + RM, len(ERASED)
    nblocks = SMALL_BLOCKS if form == "small" else T["nblocks"]
    frames_h = T["frames"] if layout == "arena" else T["frames"][::-1]
    store = torch.from_numpy(np.ascontiguousarray(frames_h)).to("cuda:0")
    frame = (lambda i: store[i]) if layout == "arena" else (lambda i: store[n - 1 - i])
    ptrs = [0 if i in ERASED else frame(i).data_ptr() for i in range(n)]
    want = [int(i in ERASED) for i in range(n)]
    pitch = round_up(S, 16) + GUARD
    out = torch.full((nblocks * r, pitch), FILL, dtype=torch.uint8, device="cuda:0")
    dig = torch.full((nblocks, RK + r, 32), FILL, dtype=torch.uint8, device="cuda:0")
    cor = torch.zeros((nblocks, RK), dtype=torch.uint8, device="cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    c = mb.Codec(RK, RM, T["bs"])
    try:
        for name, v in opts.items():
            c.set_option(name, v)

        def reconstruct():
            before = form_counts(c)
            cor.zero_()
            c.reconstruct_device(ptrs, fp, nblocks, want, 0, out.data_ptr(), pitch, dig.data_ptr(), cor.data_ptr(), st)
            torch.cuda.synchronize()
            delta, last = form_delta(before, form_counts(c)), last_launch(c)
            assert delta == {form: 1}, delta
            if form == "small":
                assert (last["last_eb"], last["last_grid"], last["last_row_chunk"]) == (1, nblocks, ROW_CHUNK[r]), last
            else:
                tma = TMA_BYTEWISE if form == "dyn_bytewise" else (TMA_RUNS if layout == "arena" else TMA_PER_INPUT)
                assert (last["last_eb"], last["last_grid"], last["last_tma_mode"], last["last_direct"], last["last_row_chunk"]) == \
                       (4, num_sms, tma, int(form == "dyn_aligned"), ROW_CHUNK[r]), last
                assert ceil_div(nblocks, 4) > last["last_grid"]
            return last

        last = reconstruct()
        assert int(cor.sum().item()) == 0, "a clean frame was flagged"
        got = out.view(nblocks, r, pitch).cpu().numpy()
        assert_blocks_equal(got[:, :, :S], T["shards"][:nblocks, list(ERASED)], "rebuilt shards")
        assert (got[:, :, S:] == FILL).all(), "rebuilt rows were written past the shard end"
        hd = dig.cpu().numpy()
        assert_blocks_equal(hd[:, :RK], T["dig"][:nblocks, READERS], "reader digests")
        assert_blocks_equal(hd[:, RK:], T["dig"][:nblocks, list(ERASED)], "rebuilt-shard digests")

        if form == "small":
            b, pos = nblocks - 1, RK - 1
        else:   # block 4 * grid + 6: group grid + 1, a CTA's second group
            b, pos = 4 * last["last_grid"] + 6, 5
            assert b // 4 >= last["last_grid"] and b < nblocks
        f = frame(READERS[pos])
        assert S % 32 > 1
        for byte, flagged_want in ((32 + 32 * (S // 32), [[b, pos]]), (32 + S - 1, [[b, pos]]), (32 + S, []), (fp - 1, [])):
            f[b, byte] ^= 0x40
            reconstruct()
            f[b, byte] ^= 0x40
            flagged = torch.nonzero(cor).cpu().tolist()
            assert flagged == flagged_want, (b, byte, flagged)
    finally:
        c.close()
