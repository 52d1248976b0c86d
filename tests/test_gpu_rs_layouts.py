"""The layouts the C ABI promises for the batched Reed-Solomon encode / reconstruct calls and the Crossword distribute
beyond the 16-byte-aligned ones the rest of the suite uses (include/summerset_b200.h): payloads at any byte offset of the
arena, byte-exact stores without SS_RS_OUT_PADDED16, and SS_RS_EMIT_DATA (the data shards written into planes 0..d-1 of
the shard store).  A caller holding bincode-packed request batches and exact-length shard buffers relies on all three.

Method, for every case:
  * the payload arena is random bytes, gaps between payloads included, so a kernel that lets bytes past a payload's end
    into a shard changes the result;
  * the output buffer starts as random canary bytes; the expected buffer is a copy of the canary with the CPU oracle's
    writes applied (plus the zero padding SS_RS_OUT_PADDED16 defines), and the GPU's buffer must equal it over EVERY byte:
    slots, padding, the gaps between slots and the planes a call must leave alone, in one comparison;
  * rs.last_kernel() pins the kernel each case reaches.
"""
import numpy as np
import pytest
import torch

from summerset_b200 import workloads as wl
from summerset_b200._lib import check
from summerset_b200.api import ReedSolomon, cw_slot_pitch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PADDED16, EMIT_DATA = 1, 2          # SS_RS_OUT_PADDED16, SS_RS_EMIT_DATA
FLAGS = [PADDED16, PADDED16 | EMIT_DATA, 0, EMIT_DATA]
FLAG_IDS = ["padded", "padded+emit", "exact", "exact+emit"]


# ---------------------------------------------------------------------------------------------
# layouts and expectations
# ---------------------------------------------------------------------------------------------
def _lengths(rng, d):
    """A ragged batch's payload lengths, shuffled: null codewords; lengths around d and 16*d; shard lengths just under, at
    and over 1024 bytes (64 unmasked 16-byte columns, where rs32_encode_ragged_kernel starts pairing columns); long
    payloads; the cfg-4 sizes; random ones."""
    edges = [0, 0, 1, 2, d - 1, d, d + 1, 15, 16, 17, 16 * d - 1, 16 * d, 16 * d + 1, 511, 512,
             1023 * d, 1024 * d - 1, 1024 * d, 1024 * d + 1, 4096, 9001, 65536 + 3]
    lens = np.concatenate([edges, wl.CFG4_SIZES, rng.integers(1, 3001, 200)]).astype(np.uint32)
    rng.shuffle(lens)
    return lens


def _shard_lens(lens, d):
    return (lens.astype(np.int64) + d - 1) // d


def _ranges(starts, counts):
    """flat indices of the byte ranges [starts[i], starts[i] + counts[i])"""
    starts = np.asarray(starts, dtype=np.int64)
    counts = np.asarray(counts, dtype=np.int64)
    first = np.cumsum(counts) - counts
    return np.arange(int(counts.sum()), dtype=np.int64) + np.repeat(starts - first, counts)


def _arena(rng, lens, lead=16, slack=32):
    """Payloads back to back, each after a random gap of 0..31 bytes, so they start at every byte offset mod 16.  The
    kernels may load up to 15 bytes either side of a payload: `lead` and `slack` keep those loads inside the arena."""
    gaps = rng.integers(0, 32, len(lens))
    ends = np.cumsum(lens.astype(np.int64) + gaps)
    data_off = lead + ends - lens.astype(np.int64)
    assert len(np.unique(data_off % 16)) == 16
    arena = rng.integers(0, 256, lead + int(ends[-1]) + slack, dtype=np.uint8)
    return arena, data_off.astype(np.uint64)


def _slots(rng, L, padded):
    """One shard slot per codeword in each plane -> (offsets, plane_stride).  Padded: 16-byte aligned offsets with
    capacity round_up(L,16) and 0..2 spare vectors between slots, plane_stride a multiple of 16.  Byte-exact: L-byte slots
    packed after odd gaps of 1..15 bytes from an odd start, odd plane_stride."""
    if padded:
        size = (L + 15) // 16 * 16 + 16 * rng.integers(0, 3, len(L))
        start = 16
    else:
        size = L + 2 * rng.integers(0, 8, len(L)) + 1
        start = 19
    off = start + np.cumsum(size) - size
    stride = start + int(size.sum()) + 32
    stride = (stride + 15) // 16 * 16 if padded else stride | 1
    return off.astype(np.uint64), stride


def _split(oracle, arena, data_off, lens, g, d):
    """the d data shards of codeword g (oracle.cw_split: contiguous split of the zero-padded payload)"""
    o = int(data_off[g])
    return oracle.cw_split(arena[o:o + int(lens[g])].tobytes(), d)


def _expect_encode(oracle, d, p, canary, arena, data_off, lens, par_off, plane_stride, flags):
    """What an encode must leave in the (d+p)-plane buffer `canary` [d+p, plane_stride]: the oracle's parity in planes
    d.., the data shards in planes 0..d-1 with SS_RS_EMIT_DATA, zeros over [L, round_up(L,16)) of every slot written with
    SS_RS_OUT_PADDED16, and the canary everywhere else."""
    want = canary.copy()
    L = _shard_lens(lens, d)
    live = np.nonzero(lens)[0]
    first = 0 if flags & EMIT_DATA else d
    if flags & PADDED16:
        pad = _ranges(par_off[live].astype(np.int64) + L[live], (L[live] + 15) // 16 * 16 - L[live])
        want[first:, pad] = 0
    oracle.rs_encode_batch(d, p, arena, data_off, lens, want[d:].reshape(-1), plane_stride, par_off)
    if flags & EMIT_DATA:
        for g in live:
            o = int(par_off[g])
            want[:d, o:o + L[g]] = _split(oracle, arena, data_off, lens, g, d)
    return want


def _assert_same(got, want, slot_off=None, lens=None):
    """whole-buffer equality; on failure names the first differing byte and the codeword whose slot region holds it"""
    if np.array_equal(got, want):
        return
    bad = np.argwhere(got != want)
    j, pos = (int(x) for x in bad[0])
    msg = f"{len(bad)} bytes differ; first in plane {j} at byte {pos}: got {got[j, pos]:#04x}, want {want[j, pos]:#04x}"
    if slot_off is not None:
        order = np.argsort(slot_off, kind="stable")
        k = int(np.searchsorted(slot_off[order], pos, side="right")) - 1
        if k >= 0:
            g = int(order[k])
            msg += f" (slot region of codeword {g}: data_len {int(lens[g])}, slot offset {int(slot_off[g])})"
    pytest.fail(msg)


def _dev(a, dtype):
    """A device copy.  Hold the returned tensor until the kernel has run: a raw data_ptr() does not keep it alive, and the
    caching allocator hands a dropped tensor's memory to the next allocation."""
    return torch.from_numpy(np.ascontiguousarray(a).astype(dtype)).to(DEV)


# ---------------------------------------------------------------------------------------------
# ss_rs_encode_batch_dev: unaligned payloads, padded and byte-exact slots, with and without SS_RS_EMIT_DATA
# ---------------------------------------------------------------------------------------------
# (d, p, variant, kernel): RS(3,2); every dispatch_d capacity of the Horner kernel (2, 3, 4, 6, 8); every dispatch_p case
# of the bit-plane kernel (p = 1, 2, 3, 4, 5-6, 7-8), which also serves d > 8; the bit-plane kernel forced by variant 5
ENCODE_CODES = [
    (3, 2, 0, "rs32_encode_ragged_kernel"),
    (2, 1, 0, "horner_encode_ragged_kernel"), (3, 1, 0, "horner_encode_ragged_kernel"),
    (4, 3, 0, "horner_encode_ragged_kernel"), (5, 4, 0, "horner_encode_ragged_kernel"),
    (6, 4, 0, "horner_encode_ragged_kernel"), (7, 2, 0, "horner_encode_ragged_kernel"),
    (8, 8, 0, "horner_encode_ragged_kernel"),
    (10, 1, 0, "generic_encode_ragged_kernel"), (11, 2, 0, "generic_encode_ragged_kernel"),
    (17, 3, 0, "generic_encode_ragged_kernel"), (20, 4, 0, "generic_encode_ragged_kernel"),
    (9, 6, 0, "generic_encode_ragged_kernel"), (12, 8, 0, "generic_encode_ragged_kernel"),
    (24, 8, 0, "generic_encode_ragged_kernel"),
    (4, 3, 5, "generic_encode_ragged_kernel"),
]


@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
@pytest.mark.parametrize("d,p,variant,kernel", ENCODE_CODES)
def test_encode_batch_unaligned_payloads(ctx, oracle, d, p, variant, kernel, flags):
    rng = np.random.default_rng(7000 + 100 * d + 10 * p + variant + flags)
    rs = ReedSolomon(ctx, d, p)
    rs.set_variant(variant)
    lens = _lengths(rng, d)
    n = len(lens)
    arena, data_off = _arena(rng, lens)
    par_off, ps = _slots(rng, _shard_lens(lens, d), flags & PADDED16)
    canary = rng.integers(0, 256, (d + p, ps), dtype=np.uint8)
    buf = torch.from_numpy(canary.copy()).to(DEV)
    a, do, ln, po = _dev(arena, np.uint8), _dev(data_off, np.int64), _dev(lens, np.int32), _dev(par_off, np.int64)
    # parity = plane d of the (d+p)-plane store, as SS_RS_EMIT_DATA defines it; without the flag planes 0..d-1 stay canary
    check(ctx.lib.ss_rs_encode_batch_dev(rs.h, a.data_ptr(), do.data_ptr(), ln.data_ptr(), n, buf.data_ptr() + d * ps, ps,
                                         po.data_ptr(), flags))
    torch.cuda.synchronize()
    assert rs.last_kernel() == kernel
    want = _expect_encode(oracle, d, p, canary, arena, data_off, lens, par_off, ps, flags)
    _assert_same(buf.cpu().numpy(), want, par_off, lens)


# ---------------------------------------------------------------------------------------------
# ss_rs_encode_uniform_dev on the flat kernels: odd payload stride, odd output base in the byte-exact layout
# ---------------------------------------------------------------------------------------------
UNIFORM_CODES = [
    (3, 2, 1, "rs32_encode_uniform_kernel"),
    (4, 3, 1, "horner_encode_uniform_kernel"),
    (9, 6, 0, "generic_encode_uniform_kernel"),
    (17, 3, 0, "generic_encode_uniform_kernel"),
]


@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
@pytest.mark.parametrize("d,p,variant,kernel", UNIFORM_CODES)
def test_encode_uniform_flat_kernels_odd_stride(ctx, oracle, d, p, variant, kernel, flags):
    rng = np.random.default_rng(8000 + 100 * d + 10 * p + flags)
    rs = ReedSolomon(ctx, d, p)
    rs.set_variant(variant)
    n, lead = 37, 21                                       # codeword g starts at byte 21 + g * stride of the arena
    for data_len in (1, d + 1, 16 * d - 1, 1000, 4099):
        stride = (data_len + 7) | 1
        arena = rng.integers(0, 256, lead + n * stride + 32, dtype=np.uint8)
        data_off = (lead + np.arange(n) * stride).astype(np.uint64)
        lens = np.full(n, data_len, dtype=np.uint32)
        L = -(-data_len // d)
        if flags & PADDED16:
            ss, base = (L + 15) // 16 * 16 + 16, 16
        else:
            ss, base = L + 3, 21
        par_off = (base + np.arange(n) * ss).astype(np.uint64)
        ps = base + n * ss + 32
        ps = (ps + 15) // 16 * 16 if flags & PADDED16 else ps | 1
        canary = rng.integers(0, 256, (d + p, ps), dtype=np.uint8)
        buf = torch.from_numpy(canary.copy()).to(DEV)
        a = _dev(arena, np.uint8)
        check(ctx.lib.ss_rs_encode_uniform_dev(rs.h, a.data_ptr() + lead, stride, data_len, n,
                                               buf.data_ptr() + d * ps + base, ps, ss, flags))
        torch.cuda.synchronize()
        assert rs.last_kernel() == kernel, data_len
        want = _expect_encode(oracle, d, p, canary, arena, data_off, lens, par_off, ps, flags)
        _assert_same(buf.cpu().numpy(), want, par_off, lens)


# ---------------------------------------------------------------------------------------------
# ss_rs_reconstruct_batch_dev, byte-exact: odd slot offsets and plane stride, every present mask in one shuffled batch
# ---------------------------------------------------------------------------------------------
RECON_CODES = [
    (1, 1, 0, "rs_reconstruct_small_kernel(smem programs)"),
    (2, 1, 0, "rs_reconstruct_small_kernel(smem programs)"),
    (3, 2, 0, "rs_reconstruct_small_kernel(smem programs)"),
    (4, 3, 0, "rs_reconstruct_small_kernel"),              # compact programs above 40 KB: read from global memory
    (4, 4, 0, "rs_reconstruct_small_kernel"),
    (5, 4, 0, "horner_reconstruct_kernel"), (6, 4, 0, "horner_reconstruct_kernel"),
    (7, 2, 0, "horner_reconstruct_kernel"), (8, 4, 0, "horner_reconstruct_kernel"),
    (9, 2, 0, "generic_reconstruct_kernel"), (10, 2, 0, "generic_reconstruct_kernel"),
    (3, 2, 5, "generic_reconstruct_kernel"), (3, 2, 8, "horner_reconstruct_kernel"),
]


@pytest.mark.parametrize("data_only", [True, False], ids=["data_only", "full"])
@pytest.mark.parametrize("d,p,variant,kernel", RECON_CODES)
def test_reconstruct_batch_byte_exact_every_mask(ctx, oracle, d, p, variant, kernel, data_only):
    t = d + p
    rng = np.random.default_rng(9000 + 100 * d + 10 * p + variant)
    rs = ReedSolomon(ctx, d, p)
    rs.set_variant(variant)
    # every present mask at least twice, shuffled, so that warps walk mixed patterns
    present = np.tile(np.arange(1 << t, dtype=np.uint32), max(2, 4096 >> t))
    rng.shuffle(present)
    n = len(present)
    mix = _lengths(rng, d)
    lens = np.concatenate([mix, rng.integers(1, 3001, n - len(mix))]).astype(np.uint32)
    rng.shuffle(lens)
    L = _shard_lens(lens, d)
    arena, data_off = _arena(rng, lens)
    off, ps = _slots(rng, L, padded=False)
    # intact codewords in their slots, canary bytes around them
    intact = rng.integers(0, 256, (t, ps), dtype=np.uint8)
    live = np.nonzero(lens)[0]
    for g in live:
        o = int(off[g])
        intact[:d, o:o + L[g]] = _split(oracle, arena, data_off, lens, g, d)
    oracle.rs_encode_batch(d, p, arena, data_off, lens, intact[d:].reshape(-1), ps, off)
    # missing shards hold garbage over their L bytes only
    damaged = intact.copy()
    for j in range(t):
        miss = ((present >> j) & 1) == 0
        idx = _ranges(off[miss].astype(np.int64), L[miss])
        damaged[j, idx] = rng.integers(0, 256, len(idx), dtype=np.uint8)
    want = damaged.copy()
    st_want = oracle.rs_reconstruct_batch(d, p, want.reshape(-1), ps, off, lens, present, data_only)

    sh = torch.from_numpy(damaged.copy()).to(DEV)
    st = torch.full((n,), 12345, dtype=torch.int32, device=DEV)
    do, ln, pr = _dev(off, np.int64), _dev(lens, np.int32), _dev(present, np.int32)
    check(ctx.lib.ss_rs_reconstruct_batch_dev(rs.h, sh.data_ptr(), ps, do.data_ptr(), ln.data_ptr(), pr.data_ptr(), n,
                                              1 if data_only else 0, st.data_ptr(), 0))
    torch.cuda.synchronize()
    assert rs.last_kernel() == kernel
    got = sh.cpu().numpy()
    st = st.cpu().numpy()

    # status: SS_ERR_INVALID_ARG for null codewords, SS_ERR_TOO_FEW_SHARDS_PRESENT below d shards, else 0
    npresent = sum(((present >> j) & 1).astype(np.int64) for j in range(t))
    st_expect = np.where(lens == 0, -20, np.where(npresent < d, -10, 0))
    assert (st_want == st_expect).all()
    bad = np.nonzero(st != st_want)[0]
    assert len(bad) == 0, f"status of codeword {bad[0]} (present {present[bad[0]]:#x}): {st[bad[0]]}, want {st_want[bad[0]]}"
    # every byte: regenerated slots, present shards, codewords with too few shards, gaps and guard bands
    _assert_same(got, want, off, lens)
    # and the regenerated bytes are the intact codeword's, so the oracle and the kernels cannot drift together
    for j in range(d if data_only else t):
        regen = (st == 0) & (((present >> j) & 1) == 0)
        idx = _ranges(off[regen].astype(np.int64), L[regen])
        assert np.array_equal(got[j, idx], intact[j, idx]), j


# ---------------------------------------------------------------------------------------------
# ss_crossword_distribute_dev: unaligned payloads into 32-byte-pitch replica slots
# ---------------------------------------------------------------------------------------------
# (population, d, p, variant, kernel)
CW_CASES = [
    (5, 3, 2, 0, "rs32_crossword_distribute_kernel<1>"),
    (5, 3, 2, 6, "rs32_crossword_distribute_kernel<8,dynamic>"),
    (5, 3, 2, 7, "rs32_crossword_distribute_kernel<4,dynamic>"),
    (5, 6, 4, 0, "crossword_distribute_generic_kernel"),
    (5, 6, 4, 1 << 11, "crossword_distribute_generic_kernel"),
    (7, 4, 3, 0, "crossword_distribute_generic_kernel<static>"),
    (7, 4, 3, 1 << 11, "crossword_distribute_generic_kernel"),
]


@pytest.mark.parametrize("n_rep,d,p,variant,kernel", CW_CASES)
def test_crossword_distribute_unaligned_payloads(ctx, oracle, n_rep, d, p, variant, kernel):
    T = d + p
    dj = T // n_rep
    rng = np.random.default_rng(9500 + 100 * n_rep + 10 * d + (variant & 15) + (variant >> 11))
    rs = ReedSolomon(ctx, d, p)
    rs.set_variant(variant)
    lens = _lengths(rng, d)
    n = len(lens)
    arena, data_off = _arena(rng, lens)
    choices = np.arange(dj, d + 1, dj)                     # the spr values the assignment policy can pick
    spr = choices[rng.integers(0, len(choices), n)].astype(np.uint8)
    L = _shard_lens(lens, d)
    lp = cw_slot_pitch(L)
    slot_bytes = spr.astype(np.int64) * lp
    rep_off = 32 + np.cumsum(slot_bytes) - slot_bytes
    total = (32 + int(slot_bytes.sum()) + 64 + 31) // 32 * 32
    canary = rng.integers(0, 256, (n_rep, total), dtype=np.uint8)
    logs = torch.from_numpy(canary.copy()).to(DEV)
    args = (_dev(arena, np.uint8), _dev(data_off, np.int64), _dev(lens, np.int32), _dev(spr, np.uint8), _dev(rep_off, np.int64))
    rs.crossword_distribute(*args, [logs[r].data_ptr() for r in range(n_rep)])
    torch.cuda.synchronize()
    assert rs.last_kernel() == kernel
    # expected logs: the canary, with replica r's slot k of codeword g = shard (r*dj + k) mod T, zero past L
    par_off = (np.cumsum(L) - L).astype(np.uint64)
    par = np.zeros((p, int(L.sum()) + 1), dtype=np.uint8)
    oracle.rs_encode_batch(d, p, arena, data_off, lens, par.reshape(-1), par.shape[1], par_off)
    want = canary.copy()
    asg = {int(s): oracle.cw_brr_assignment(n_rep, T, int(s)) for s in choices}
    for g in np.nonzero(lens)[0]:
        Lg, lpg, k, ro = int(L[g]), int(lp[g]), int(spr[g]), int(rep_off[g])
        po = int(par_off[g])
        shards = np.concatenate([_split(oracle, arena, data_off, lens, g, d), par[:, po:po + Lg]])
        for r in range(n_rep):
            held = [(r * dj + kk) % T for kk in range(k)]
            assert sum(1 << j for j in held) == int(asg[k][r])        # the reference's assignment, bit for bit
            slots = want[r, ro:ro + k * lpg].reshape(k, lpg)
            slots[:, :Lg] = shards[held]
            slots[:, Lg:] = 0
    _assert_same(logs.cpu().numpy(), want, rep_off, lens)
