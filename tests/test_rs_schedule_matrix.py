"""The batched reconstruct (ss_rs_reconstruct_uniform_dev / ss_rs_reconstruct_batch_dev) and the Crossword distribute
(ss_crossword_distribute_dev) at every kernel instance their launchers reach, past the first pass of every grid.

All of these kernels walk a batch with a grid-stride loop and fetch the next codeword's metadata (present mask, length,
offset) one grid stride ahead; the dynamic distribute kernels take runs of codewords from a counter and pool the short
codewords of a run into shared column passes.  A mistake in any of those schemes leaves the first grid pass correct and
corrupts only the codewords after it, so every instance here runs at batch sizes just below, at, just above and several
times the number of codewords its grid covers in one pass, computed from ctx.sm_count:
  * ragged reconstruct / distribute kernels (ragged_grid): sm_count * 32 CTAs of 8 warps, a warp per codeword;
  * rs32_reconstruct_row_kernel: sm_count * per_sm * waves CTAs, a CTA per codeword (waves from variant bits 5-7);
  * dynamic distribute kernels: sm_count * 3 CTAs of 8 warps, RUN codewords per take from the counter.

Expected values come from the CPU oracle (oracle/pyoracle.py), and every output buffer is compared over every byte:
slots, the padding a padded call writes as zeros, the slack between slots, planes a data-only call must leave alone,
replica-log slots past spr, and the gaps.  Buffers start as random canary bytes; missing shards hold garbage; the status
arrays sit between guard words; a random half of the present masks carry garbage above bit d+p, which both launchers
ignore.  Batches of 10^5..10^6 codewords are compared on the device (torch.equal over the whole buffer, the device form
of np.array_equal); a uniform batch is assembled on the device from a table of prototype codewords, each under every
present mask, so that only the table goes through the oracle.
"""
import functools
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from summerset_b200._lib import SS_ERR_INVALID_ARG, SS_ERR_UNSUPPORTED, SS_OK, check
from summerset_b200.api import Context, ReedSolomon, cw_slot_pitch
from tests.test_gpu_rs_layouts import _arena, _ranges, _shard_lens, _slots

DEV = "cuda:0"
PADDED16 = 1
PAIR = 1 << 16                  # variant bit 16: two columns per lane in rs_reconstruct_small_kernel
GUARD = 16                      # guard words either side of a status array
TAIL = 8192                     # canary bytes after the last plane of a ragged batch
SENTINEL = 0x5A5A5A5A
ROOT = Path(__file__).resolve().parent.parent

# every name the reconstruct and distribute launchers can report through rs.last_kernel()
RECON_KERNELS = {
    "rs32_reconstruct_row_kernel",
    "rs_reconstruct_small_kernel(smem programs)", "rs_reconstruct_small_kernel",
    "horner_reconstruct_kernel", "generic_reconstruct_kernel",
}
DIST_KERNELS = {
    "rs32_crossword_distribute_kernel<1>", "rs32_crossword_distribute_kernel<8,dynamic>",
    "rs32_crossword_distribute_kernel<4,dynamic>",
    "crossword_distribute_generic_kernel<static>", "crossword_distribute_generic_kernel",
}
REACHED = set()                 # last_kernel() of every matrix case that ran
DONE = set()                    # matrix cases that ran to the end


def _pad16(L):
    return (L + 15) // 16 * 16


def _ragged_cap(ctx):
    """codewords one pass of ragged_grid covers: sm_count * 32 CTAs of 8 warps, a warp per codeword"""
    return ctx.sm_count * 32 * 8


def _grid_edges(cap, tail=77):
    return [cap - 1, cap, cap + 1, 3 * cap + tail]


def _status_buf(n):
    return torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int32, device=DEV)


def _status_want(st, n):
    """the status array after a call on the first n codewords: st[:n] between untouched guard / sentinel words"""
    want = np.full(len(st) + 2 * GUARD, SENTINEL, dtype=np.int64).astype(np.int32)
    want[GUARD:GUARD + n] = st[:n]
    return torch.from_numpy(want).to(DEV)


def _same(got, want, what):
    """every byte equal, on the device; on failure the number of differing bytes and the first one"""
    if torch.equal(got, want):
        return
    bad = torch.nonzero(got != want)
    first = tuple(int(x) for x in bad[0])
    pytest.fail(f"{what}: {bad.shape[0]} elements differ; first at {first}: got {int(got[first])}, want {int(want[first])}")


def _garbage_high_bits(rng, present, t):
    """a random half of the masks with random bits at and above bit t (the launchers mask them off)"""
    hi = (rng.integers(1, 1 << (32 - t), len(present), dtype=np.int64) << t) & 0xFFFFFFFF
    return np.where(rng.integers(0, 2, len(present)) == 1, present | hi, present).astype(np.uint32)


def _data_shards_into(planes, arena, data_off, lens, d, off):
    """oracle.cw_split for a whole batch: data shard i of codeword g = payload bytes [i*L, (i+1)*L), zero past the
    payload, written to planes[i, off[g] .. +L)"""
    L = _shard_lens(lens, d)
    for i in range(d):
        cnt = np.clip(lens.astype(np.int64) - i * L, 0, L)
        planes[i, _ranges(off.astype(np.int64), cnt)] = arena[_ranges(data_off.astype(np.int64) + i * L, cnt)]
        planes[i, _ranges(off.astype(np.int64) + cnt, L - cnt)] = 0


# ---------------------------------------------------------------------------------------------
# the names the launchers report (no device)
# ---------------------------------------------------------------------------------------------
def _launcher_names(fn):
    src = (ROOT / "summerset_b200" / "csrc" / "rs_kernels.cu").read_text()
    m = re.search(r"\nint " + fn + r"\(.*?\n}\n", src, re.S)
    assert m, fn
    names = set()
    for stmt in re.findall(r"last_kernel\s*=\s*([^;]+);", m.group(0)):
        names.update(re.findall(r'"([^"]+)"', stmt))
    return names


def test_kernel_name_tables_match_the_launchers():
    """RECON_KERNELS / DIST_KERNELS are exactly what the launchers can report, so the reach check at the end of this
    file covers every instance family"""
    assert _launcher_names("launch_rs_reconstruct") | _launcher_names("launch_rs_reconstruct_uniform") == RECON_KERNELS
    assert _launcher_names("launch_crossword_distribute") == DIST_KERNELS


def test_batch_split_matches_oracle(oracle):
    """the vectorised split used to build intact codewords equals oracle.cw_split codeword by codeword"""
    rng = np.random.default_rng(1)
    for d in (1, 2, 3, 5, 9):
        lens = np.array([0, 1, d - 1 or 1, d, d + 1, 15, 16, 17, 16 * d - 1, 16 * d + 1, 1000, 4097], dtype=np.uint32)
        lens = np.tile(lens, 8)
        arena, data_off = _arena(rng, lens)
        L = _shard_lens(lens, d)
        off = (np.cumsum(L) - L).astype(np.uint64)
        planes = rng.integers(0, 256, (d, int(L.sum()) + 1), dtype=np.uint8)
        _data_shards_into(planes, arena, data_off, lens, d, off)
        for g in range(len(lens)):
            o, dl = int(data_off[g]), int(lens[g])
            want = oracle.cw_split(arena[o:o + dl].tobytes(), d) if dl else np.zeros((d, 0), np.uint8)
            assert np.array_equal(planes[:, int(off[g]):int(off[g]) + int(L[g])], want), (d, g)


def test_prototype_tables_match_oracle(oracle):
    """each entry of the uniform prototype table is what the oracle makes of that codeword under that mask"""
    d, p, data_len, ss = 3, 2, 50, 48
    tab = _proto_tables(oracle, d, p, data_len, ss, 3, 11)
    L = 17
    t, M = d + p, 1 << (d + p)
    for c in (0, 5, M + 7, 2 * M + 31, 3 * M - 1):
        m = c % M
        planes = np.ascontiguousarray(tab.dmg[c])
        for data_only in (True, False):
            got = planes.copy()
            st = oracle.rs_reconstruct_batch(d, p, got.reshape(-1), ss, np.zeros(1, np.uint64),
                                             np.array([data_len], np.uint32), np.array([m], np.uint32), data_only)
            assert st[0] == tab.st[data_only][c]
            outs = range(d) if data_only else range(t)
            for j in range(t):
                if st[0] == 0 and not (m >> j) & 1 and j in outs:
                    got[j, L:_pad16(L)] = 0
            assert np.array_equal(got, tab.want[data_only][c]), (c, data_only)
        # present shards: data shards of the prototype's payload, zero padding, canary slack
        for j in range(t):
            if (m >> j) & 1:
                assert not tab.dmg[c, j, L:_pad16(L)].any()


# ---------------------------------------------------------------------------------------------
# uniform batches assembled on the device from prototype codewords
# ---------------------------------------------------------------------------------------------
class _Protos:
    pass


@functools.lru_cache(maxsize=2)
def _proto_tables(oracle, d, p, data_len, ss, K, seed):
    """K random codewords of data_len bytes in ss-byte slots, each under every present mask m: entry c = k * 2^(d+p) + m.
    dmg[c]: the (d+p, ss) slot images a caller hands in (present shards intact with zero padding, missing shards
    garbage over their round_up(L,16) bytes, canary slack); want[data_only][c]: the images after the call; st[..][c]:
    the status."""
    rng = np.random.default_rng(seed)
    t, M = d + p, 1 << (d + p)
    L = -(-data_len // d)
    L16 = _pad16(L)
    pay = rng.integers(0, 256, K * data_len, dtype=np.uint8)
    lens = np.full(K, data_len, dtype=np.uint32)
    pay_off = (np.arange(K) * data_len).astype(np.uint64)
    slot_off = (np.arange(K) * ss).astype(np.uint64)
    planes = rng.integers(0, 256, (t, K * ss), dtype=np.uint8)
    _data_shards_into(planes, pay, pay_off, lens, d, slot_off)
    oracle.rs_encode_batch(d, p, pay, pay_off, lens, planes[d:].reshape(-1), K * ss, slot_off)
    intact = planes.reshape(t, K, ss).transpose(1, 0, 2).copy()
    intact[:, :, L:L16] = 0
    C = K * M
    m = np.arange(C) % M
    miss = ((m[:, None] >> np.arange(t)[None, :]) & 1) == 0
    dmg = np.repeat(intact, M, axis=0)
    garbage = rng.integers(0, 256, (C, t, L16), dtype=np.uint8)
    dmg[:, :, :L16] = np.where(miss[:, :, None], garbage, dmg[:, :, :L16])
    tab = _Protos()
    tab.dmg, tab.want, tab.st, tab.M, tab.L = dmg, {}, {}, M, L
    for data_only in (True, False):
        flat = dmg.transpose(1, 0, 2).copy()
        st = oracle.rs_reconstruct_batch(d, p, flat.reshape(-1), C * ss, (np.arange(C) * ss).astype(np.uint64),
                                         np.full(C, data_len, np.uint32), m.astype(np.uint32), data_only)
        want = flat.transpose(1, 0, 2).copy()
        regen = (st == 0)[:, None] & miss & ((np.arange(t) < d)[None, :] if data_only else True)
        want[:, :, L:L16] = np.where(regen[:, :, None], 0, want[:, :, L:L16])
        tab.want[data_only], tab.st[data_only] = want, st
    return tab


class _Uniform:
    """n_max codewords of one prototype table in a (d+p)-plane device buffer: codeword g's shard j at
    j*ps + g*ss, a canary tail after the last slot of each plane"""

    def __init__(self, tab, d, p, data_len, ss, n_max, seed):
        rng = np.random.default_rng(seed)
        t = d + p
        self.t, self.data_len, self.ss, self.n_max, self.tab = t, data_len, ss, n_max, tab
        self.ps = n_max * ss + 64
        comb = rng.integers(0, len(tab.dmg), n_max)
        self.comb = torch.from_numpy(comb).to(DEV)
        self.present = torch.from_numpy(_garbage_high_bits(rng, (comb % tab.M).astype(np.uint32), t).view(np.int32)).to(DEV)
        self.buf0 = torch.empty((t, self.ps), dtype=torch.uint8, device=DEV)
        self.buf0[:, n_max * ss:] = torch.from_numpy(rng.integers(0, 256, (t, 64), dtype=np.uint8)).to(DEV)
        self._fill(self.buf0, tab.dmg)
        self.comb_np = comb

    def _fill(self, buf, table):
        dev = torch.from_numpy(table).to(DEV)
        step = 1 << 18
        for a in range(0, self.n_max, step):
            b = min(self.n_max, a + step)
            buf[:, a * self.ss:b * self.ss] = dev[self.comb[a:b]].permute(1, 0, 2).reshape(self.t, (b - a) * self.ss)

    def want(self, data_only):
        w = torch.empty((self.t, self.n_max * self.ss), dtype=torch.uint8, device=DEV)
        self._fill(w, self.tab.want[data_only])
        return w, self.tab.st[data_only][self.comb_np]

    def run(self, rs, n, data_only, want, st_all, kernel, label):
        work = self.buf0.clone()
        st = _status_buf(self.n_max)
        check(rs.lib.ss_rs_reconstruct_uniform_dev(rs.h, work.data_ptr(), self.ps, self.ss, self.data_len, self.present.data_ptr(),
                                                   n, 1 if data_only else 0, st.data_ptr() + 4 * GUARD))
        torch.cuda.synchronize()
        assert rs.last_kernel() == kernel, label
        REACHED.add(kernel)
        _same(st, _status_want(st_all, n), f"{label}: status")
        cut = n * self.ss
        _same(work[:, :cut], want[:, :cut], f"{label}: slots of the batch")
        _same(work[:, cut:], self.buf0[:, cut:], f"{label}: planes past the batch")


# ---------------------------------------------------------------------------------------------
# ss_rs_reconstruct_uniform_dev on RS(3,2): rs32_reconstruct_row_kernel at every wave setting
# ---------------------------------------------------------------------------------------------
# (data_len, threads): 32 threads (vpc <= 32), 96 threads (the 4096-byte cfg-3b payload), 160 threads (vpc = 129, the
# <256,5> build).  The slot is 16 bytes wider than round_up(L,16), so a write into the slack shows.
ROW_WIDTHS = [(45, 32), (4096, 96), (6146, 160)]
ROW_WAVES = [16, 1, 32, 4, 64, 256, 128, 8]     # launch_rs_reconstruct_uniform's table, indexed by variant bits 5-7
ROW_BUDGET = 1 << 30                             # bytes per device copy of a batch


def _row_n_values(ctx, threads, n_max):
    per_sm = min(32, 2048 // threads)
    out = {}
    for vw, waves in enumerate(ROW_WAVES):
        cap = ctx.sm_count * per_sm * waves
        out[vw] = [n for n in [1] + _grid_edges(cap) if n <= n_max]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("data_only", [True, False], ids=["data_only", "full"])
@pytest.mark.parametrize("data_len,threads", ROW_WIDTHS, ids=[f"{t}thr" for _, t in ROW_WIDTHS])
def test_uniform_rs32_row_kernel_every_wave(ctx, oracle, data_len, threads, data_only):
    """every wave setting of variant bits 5-7 x data_only x the 128- and 256-thread builds; the grid-stride loop and the
    next-mask prefetch wrap wherever the batch fits ROW_BUDGET: at every wave setting for 32-thread CTAs and up to
    16 waves for the wider ones (the wave setting changes only the grid size)"""
    d, p = 3, 2
    L = -(-data_len // d)
    vpc = -(-L // 16)
    assert min(256, (vpc + 31) // 32 * 32) == threads
    ss = _pad16(L) + 16
    per_sm = min(32, 2048 // threads)
    n_max = min(3 * ctx.sm_count * per_sm * max(ROW_WAVES) + 77, ROW_BUDGET // ((d + p) * ss))
    nv = _row_n_values(ctx, threads, n_max)
    for vw in range(8):
        if ROW_WAVES[vw] <= (16 if threads > 32 else 256):
            assert len(nv[vw]) == 5, (vw, nv[vw])     # every grid edge fits the budget
    tab = _proto_tables(oracle, d, p, data_len, ss, 61, 100 + threads)
    U = _Uniform(tab, d, p, data_len, ss, n_max, 200 + threads)
    want, st = U.want(data_only)
    rs = ReedSolomon(ctx, d, p)
    for vw in range(8):
        rs.set_variant(vw << 5)
        for n in nv[vw]:
            U.run(rs, n, data_only, want, st, "rs32_reconstruct_row_kernel", f"waves {ROW_WAVES[vw]}, n {n}")
    DONE.add(("row", threads, data_only))


# ---------------------------------------------------------------------------------------------
# ss_rs_reconstruct_uniform_dev on the fallback: uniform_meta_kernel + the ragged kernels
# ---------------------------------------------------------------------------------------------
# (d, p, variant, kernel)
FALLBACK_CODES = [
    (4, 3, 0, "rs_reconstruct_small_kernel"),
    (4, 3, PAIR, "rs_reconstruct_small_kernel"),
    (6, 4, 0, "horner_reconstruct_kernel"),
    (8, 4, 0, "horner_reconstruct_kernel"),
    (9, 3, 0, "generic_reconstruct_kernel"),
    (3, 2, 5, "generic_reconstruct_kernel"),
    (3, 2, 8, "horner_reconstruct_kernel"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("d,p,variant,kernel", FALLBACK_CODES)
def test_uniform_fallback_grid_edges(ctx, oracle, d, p, variant, kernel):
    data_len = 16 * d + 3                     # L = 17: a partial second column
    ss = 48 + 16 * (d % 2)                    # round_up(17,16) = 32 plus slack
    cap = _ragged_cap(ctx)
    tab = _proto_tables(oracle, d, p, data_len, ss, 4 if d + p <= 8 else 2, 300 + 10 * d + p)
    U = _Uniform(tab, d, p, data_len, ss, 3 * cap + 77, 400 + 10 * d + p)
    rs = ReedSolomon(ctx, d, p)
    rs.set_variant(variant)
    for data_only in (True, False):
        want, st = U.want(data_only)
        for n in [1] + _grid_edges(cap):
            U.run(rs, n, data_only, want, st, kernel, f"RS({d},{p}) v{variant:#x}, n {n}, data_only {data_only}")
    DONE.add(("fallback", d, p, variant))


@pytest.mark.gpu
def test_uniform_fallback_scratch_regrows_past_meta_grid(oracle):
    """three calls on a fresh context: n grows (the scratch for the synthesised offsets is allocated, then reallocated
    for n = 2^20 + 77, which also wraps uniform_meta_kernel's 4096 CTAs of 256 threads), then shrinks (reused)"""
    c = Context(0)
    try:
        d, p, data_len, ss = 4, 3, 61, 32
        cap = _ragged_cap(c)
        n_big = (1 << 20) + 77
        assert 4096 * 256 < n_big
        tab = _proto_tables(oracle, d, p, data_len, ss, 2, 500)
        U = _Uniform(tab, d, p, data_len, ss, n_big, 501)
        rs = ReedSolomon(c, d, p)
        want, st = U.want(False)
        for n in (cap + 1, n_big, 3 * cap + 77):
            U.run(rs, n, False, want, st, "rs_reconstruct_small_kernel", f"n {n}")
        rs.close()
    finally:
        c.close()
    DONE.add(("scratch",))


# ---------------------------------------------------------------------------------------------
# ss_rs_reconstruct_batch_dev: every ragged reconstruct instance at the grid edges
# ---------------------------------------------------------------------------------------------
LAYOUTS = {"exact": (0, 0), "padded": (PADDED16, 0), "pair": (PADDED16, PAIR)}     # (flags, variant bits)
SMALL = "rs_reconstruct_small_kernel"
SMALL_SMEM = "rs_reconstruct_small_kernel(smem programs)"
# (d, p, variant, kernel, layouts): rs_reconstruct_small_kernel<D, SMEM, PADDED, PAIR> for D = 2 (d = 1, 2), 3, 4 with the
# programs in shared memory ((32 + 128p) << (d+p) <= 40 KB) and in global memory; horner_reconstruct_kernel<2,3,4> through
# variant 8, <6> and <8> by width; generic_reconstruct_kernel<P> at every dispatch_p case
RAGGED_CODES = [
    (1, 1, 0, SMALL_SMEM, "exact padded pair"), (2, 2, 0, SMALL_SMEM, "exact padded pair"),
    (2, 8, 0, SMALL, "exact padded pair"),
    (3, 2, 0, SMALL_SMEM, "exact padded pair"), (3, 4, 0, SMALL, "exact padded pair"),
    (4, 2, 0, SMALL_SMEM, "exact padded pair"), (4, 3, 0, SMALL, "exact padded pair"),
    (2, 2, 8, "horner_reconstruct_kernel", "exact padded"), (3, 2, 8, "horner_reconstruct_kernel", "exact padded"),
    (4, 3, 8, "horner_reconstruct_kernel", "exact padded"),
    (5, 4, 0, "horner_reconstruct_kernel", "exact padded"), (6, 4, 0, "horner_reconstruct_kernel", "exact padded"),
    (7, 2, 0, "horner_reconstruct_kernel", "exact padded"), (8, 4, 0, "horner_reconstruct_kernel", "exact padded"),
    (9, 1, 0, "generic_reconstruct_kernel", "exact padded"), (10, 2, 0, "generic_reconstruct_kernel", "exact padded"),
    (9, 3, 0, "generic_reconstruct_kernel", "exact padded"), (8, 4, 5, "generic_reconstruct_kernel", "exact padded"),
    (6, 5, 5, "generic_reconstruct_kernel", "exact padded"), (6, 6, 5, "generic_reconstruct_kernel", "exact padded"),
    (4, 8, 5, "generic_reconstruct_kernel", "exact padded"), (5, 7, 5, "generic_reconstruct_kernel", "exact padded"),
]
RAGGED_CASES = [(d, p, v, k, lay) for d, p, v, k, lays in RAGGED_CODES for lay in lays.split()]


def _short_lengths(rng, n, d):
    """shuffled payload lengths: 6 % null, the edges 1, 15, 16, 17, 16d-1, 16d+1, short random ones, 2 % of 1-4 KB, so
    neighbouring warps disagree on every prefetched field"""
    edges = np.array([0, 1, 15, 16, 17, 16 * d - 1, 16 * d + 1], dtype=np.int64)
    kind = rng.integers(0, 100, n)
    lens = rng.integers(1, 40 * d, n)
    lens = np.where(kind < 42, edges[rng.integers(0, len(edges), n)], lens)
    lens = np.where(kind >= 98, rng.integers(1024, 4097, n), lens)
    return lens.astype(np.uint32)


class _Ragged:
    pass


@functools.lru_cache(maxsize=1)
def _ragged_batch(oracle, d, p, padded, n, seed):
    """n codewords (shuffled lengths, every present mask, shuffled) in their slots, the damaged buffer and, for each
    data_only mode, the buffer and status the oracle expects"""
    rng = np.random.default_rng(seed)
    t = d + p
    lens = _short_lengths(rng, n, d)
    L = _shard_lens(lens, d)
    arena, data_off = _arena(rng, lens)
    off, ps = _slots(rng, L, padded)
    planes = rng.integers(0, 256, (t, ps), dtype=np.uint8)
    _data_shards_into(planes, arena, data_off, lens, d, off)
    oracle.rs_encode_batch(d, p, arena, data_off, lens, planes[d:].reshape(-1), ps, off)
    cap_end = off.astype(np.int64) + (_pad16(L) if padded else L)
    live = lens > 0
    if padded:
        planes[:, _ranges(off[live].astype(np.int64) + L[live], _pad16(L[live]) - L[live])] = 0
    present = np.tile(np.arange(1 << t, dtype=np.uint32), -(-n // (1 << t)))[:n]
    rng.shuffle(present)
    for j in range(t):
        miss = live & (((present >> j) & 1) == 0)
        idx = _ranges(off[miss].astype(np.int64), cap_end[miss] - off[miss].astype(np.int64))
        planes[j, idx] = rng.integers(0, 256, len(idx), dtype=np.uint8)
    B = _Ragged()
    B.lens, B.L, B.off, B.ps, B.present = lens, L, off, ps, present
    B.dmg = planes
    B.want, B.st = {}, {}
    for data_only in (True, False):
        want = planes.copy()
        st = oracle.rs_reconstruct_batch(d, p, want.reshape(-1), ps, off, lens, present, data_only)
        if padded:
            for j in range(d if data_only else t):
                regen = (st == 0) & (((present >> j) & 1) == 0)
                want[j, _ranges(off[regen].astype(np.int64) + L[regen], _pad16(L[regen]) - L[regen])] = 0
        B.want[data_only], B.st[data_only] = want, st
    B.present_hi = _garbage_high_bits(rng, present, t)
    return B


@pytest.mark.gpu
@pytest.mark.parametrize("d,p,variant,kernel,layout", RAGGED_CASES)
def test_reconstruct_batch_grid_edges(ctx, oracle, d, p, variant, kernel, layout):
    flags, vbits = LAYOUTS[layout]
    cap = _ragged_cap(ctx)
    n_max = 3 * cap + 77
    B = _ragged_batch(oracle, d, p, bool(flags & PADDED16), n_max, 600 + 10 * d + p)
    rs = ReedSolomon(ctx, d, p)
    rs.set_variant(variant | vbits)
    t = d + p
    # the planes, then a canary tail as long as the longest shard: a kernel that misplaces a shard past the last plane
    # writes into the tail, where the comparison sees it, instead of past the allocation
    dmg = torch.empty(t * B.ps + TAIL, dtype=torch.uint8, device=DEV)
    dmg[:t * B.ps] = torch.from_numpy(B.dmg.reshape(-1)).to(DEV)
    dmg[t * B.ps:] = torch.from_numpy(np.random.default_rng(d).integers(0, 256, TAIL, dtype=np.uint8)).to(DEV)
    off = torch.from_numpy(B.off.astype(np.int64)).to(DEV)
    ln = torch.from_numpy(B.lens.astype(np.int32)).to(DEV)
    pr = torch.from_numpy(B.present_hi.view(np.int32)).to(DEV)
    for data_only in (True, False):
        want = torch.from_numpy(B.want[data_only]).to(DEV)
        for n in _grid_edges(cap):
            work = dmg.clone()
            st = _status_buf(n_max)
            check(ctx.lib.ss_rs_reconstruct_batch_dev(rs.h, work.data_ptr(), B.ps, off.data_ptr(), ln.data_ptr(), pr.data_ptr(),
                                                      n, 1 if data_only else 0, st.data_ptr() + 4 * GUARD, flags))
            torch.cuda.synchronize()
            label = f"RS({d},{p}) {layout}, n {n}, data_only {data_only}"
            assert rs.last_kernel() == kernel, label
            REACHED.add(kernel)
            _same(st, _status_want(B.st[data_only], n), f"{label}: status")
            cut = int(B.off[n]) if n < n_max else B.ps        # slots are in codeword order
            planes, before = work[:t * B.ps].view(t, B.ps), dmg[:t * B.ps].view(t, B.ps)
            _same(planes[:, :cut], want[:, :cut], f"{label}: slots of the batch")
            _same(planes[:, cut:], before[:, cut:], f"{label}: slots past the batch")
            _same(work[t * B.ps:], dmg[t * B.ps:], f"{label}: tail past the last plane")
    DONE.add(("ragged", d, p, variant, layout))


# ---------------------------------------------------------------------------------------------
# present bits at and above d+p
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("d,p,variant,call", [(3, 2, 0, "uniform"), (4, 3, 0, "uniform"), (3, 2, 5, "uniform"),
                                              (4, 3, 0, "ragged"), (6, 4, 0, "ragged"), (9, 1, 0, "ragged")])
def test_present_bits_above_code_are_ignored(ctx, oracle, d, p, variant, call):
    """a present word with garbage in bits >= d+p gives the bytes and status of its low bits"""
    t = d + p
    rng = np.random.default_rng(700 + 10 * d + p + variant)
    rs = ReedSolomon(ctx, d, p)
    rs.set_variant(variant)
    n = 3000
    low = rng.integers(0, 1 << t, n).astype(np.uint32)
    for hi_bit in range(t, 32):
        low[hi_bit - t] = low[hi_bit - t] | np.uint32(1 << hi_bit)      # every high bit on its own
    high = _garbage_high_bits(rng, low & np.uint32((1 << t) - 1), t)
    high[:32 - t] = low[:32 - t]
    low &= np.uint32((1 << t) - 1)
    data_len = 16 * d + 5
    L = -(-data_len // d)
    ss = _pad16(L) + 16
    base = torch.from_numpy(rng.integers(0, 256, (t, n * ss + 64), dtype=np.uint8)).to(DEV)
    lens = torch.full((n,), data_len, dtype=torch.int32, device=DEV)
    offs = torch.arange(n, dtype=torch.int64, device=DEV) * ss
    outs = []
    for pres in (low, high):
        for data_only in (0, 1):
            work = base.clone()
            st = _status_buf(n)
            pr = torch.from_numpy(pres.view(np.int32)).to(DEV)
            if call == "uniform":
                check(ctx.lib.ss_rs_reconstruct_uniform_dev(rs.h, work.data_ptr(), work.shape[1], ss, data_len, pr.data_ptr(), n,
                                                            data_only, st.data_ptr() + 4 * GUARD))
            else:
                check(ctx.lib.ss_rs_reconstruct_batch_dev(rs.h, work.data_ptr(), work.shape[1], offs.data_ptr(), lens.data_ptr(),
                                                          pr.data_ptr(), n, data_only, st.data_ptr() + 4 * GUARD, PADDED16))
            torch.cuda.synchronize()
            outs.append((work, st))
    for i in range(2):
        _same(outs[2 + i][1], outs[i][1], f"status, data_only {i}")
        _same(outs[2 + i][0], outs[i][0], f"shards, data_only {i}")
    assert (outs[0][1][GUARD:GUARD + n].cpu().numpy() == 0).any()


# ---------------------------------------------------------------------------------------------
# refusals (CPU-side checks of the launchers; they need a device context)
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_reconstruct_refusals(ctx):
    rs = ReedSolomon(ctx, 3, 2)
    buf = torch.zeros((5, 4096), dtype=torch.uint8, device=DEV)
    pr = torch.full((64,), 7, dtype=torch.int32, device=DEV)
    st = _status_buf(64)
    sp = st.data_ptr() + 4 * GUARD
    lib, b = ctx.lib, buf.data_ptr()
    # data_len = 0: null codewords cannot be reconstructed
    assert lib.ss_rs_reconstruct_uniform_dev(rs.h, b, 4096, 32, 0, pr.data_ptr(), 8, 0, sp) == SS_ERR_INVALID_ARG
    # misaligned shard_stride, plane_stride or base; shard_stride below round_up(L,16)
    assert lib.ss_rs_reconstruct_uniform_dev(rs.h, b, 4096, 40, 60, pr.data_ptr(), 8, 0, sp) == SS_ERR_INVALID_ARG
    assert lib.ss_rs_reconstruct_uniform_dev(rs.h, b, 4088, 32, 60, pr.data_ptr(), 8, 0, sp) == SS_ERR_INVALID_ARG
    assert lib.ss_rs_reconstruct_uniform_dev(rs.h, b + 8, 4096, 32, 60, pr.data_ptr(), 8, 0, sp) == SS_ERR_INVALID_ARG
    assert lib.ss_rs_reconstruct_uniform_dev(rs.h, b, 4096, 16, 60, pr.data_ptr(), 8, 0, sp) == SS_ERR_INVALID_ARG
    # n = 0: OK, nothing written
    assert lib.ss_rs_reconstruct_uniform_dev(rs.h, b, 4096, 32, 60, pr.data_ptr(), 0, 0, sp) == SS_OK
    offs = torch.zeros(8, dtype=torch.int64, device=DEV)
    lens = torch.full((8,), 60, dtype=torch.int32, device=DEV)
    assert lib.ss_rs_reconstruct_batch_dev(rs.h, b, 4096, offs.data_ptr(), lens.data_ptr(), pr.data_ptr(), 0, 0, sp, 1) == SS_OK
    torch.cuda.synchronize()
    assert not buf.any()
    assert bool((st == SENTINEL).all())
    # padded flag with a misaligned base
    assert lib.ss_rs_reconstruct_batch_dev(rs.h, b + 4, 4096, offs.data_ptr(), lens.data_ptr(), pr.data_ptr(), 8, 0, sp,
                                           PADDED16) == SS_ERR_INVALID_ARG
    # codes with d + p > 12
    for d, p in ((9, 4), (5, 8), (12, 1), (20, 3)):
        big = ReedSolomon(ctx, d, p)
        assert lib.ss_rs_reconstruct_uniform_dev(big.h, b, 4096, 32, 60, pr.data_ptr(), 8, 0, sp) == SS_ERR_UNSUPPORTED
        assert lib.ss_rs_reconstruct_batch_dev(big.h, b, 4096, offs.data_ptr(), lens.data_ptr(), pr.data_ptr(), 8, 0, sp,
                                               0) == SS_ERR_UNSUPPORTED
        big.close()
    torch.cuda.synchronize()
    assert not buf.any()
    assert bool((st == SENTINEL).all())


# ---------------------------------------------------------------------------------------------
# ss_crossword_distribute_dev
# ---------------------------------------------------------------------------------------------
LONG_MIN = 3074       # the shortest RS(3,2) payloads from here on have min(len - 2L, L) >= 1024 bytes (64 columns)


def _dyn_run_lengths(rng, n, run):
    """n payload lengths for RS(3,2), built run by run (runs of `run` consecutive codewords, as the dynamic kernels take
    them): all long (>= 64 unmasked columns: min(len - 2L, L) >= 1024), all short, all null, and mixed runs whose short
    codewords pool to 30, 32, 34 or more than 64 columns.  A short codeword pools 2 * ceil(L/32) columns (its slot pitch
    is round_up(L,32)), so pooled totals are even."""
    def short_len(cols):                      # a payload whose shard pools `cols` (even) columns
        c = cols // 2
        Lh = int(rng.integers(32 * (c - 1) + 1, 32 * c + 1))
        return max(1, 3 * Lh - int(rng.integers(0, 3)))

    def split(total, k):                      # k even column counts in [2, 60] summing to about total
        extra = rng.multinomial(total // 2 - k, np.ones(k) / k)
        return [2 * min(30, 1 + int(e)) for e in extra]

    out = []
    kinds = ["long"] + ["short"] * 5 + ["null"] * 2 + ["mix30", "mix32", "mix34", "mixbig"] * 2
    while len(out) < n:
        kind = kinds[int(rng.integers(0, len(kinds)))]
        if kind == "long":
            r = [int(x) for x in rng.integers(LONG_MIN, 3600, run)]
        elif kind == "short":
            r = [short_len(2 * int(x)) for x in rng.integers(1, 12, run)]
        elif kind == "null":
            r = [0] * run
        else:
            total = {"mix30": 30, "mix32": 32, "mix34": 34, "mixbig": int(rng.integers(33, 41)) * 2}[kind]
            nshort = run - 2
            r = [short_len(c) for c in split(total, nshort)] + [0, int(rng.integers(LONG_MIN, 3600))]
            rng.shuffle(r)
        out += r
    return np.array(out[:n], dtype=np.uint32)


class _Dist:
    pass


def _dist_batch(oracle, d, p, n_rep, lens, seed):
    """a ragged batch at every byte offset mod 16, spr in 1..d, 16-byte aligned replica slots with random 0/16-byte gaps
    between codewords, canary logs and the logs the oracle expects"""
    rng = np.random.default_rng(seed)
    T, n = d + p, len(lens)
    dj = T // n_rep
    arena, data_off = _arena(rng, lens)
    spr = rng.integers(1, d + 1, n).astype(np.uint8)
    L = _shard_lens(lens, d)
    lp = cw_slot_pitch(L)
    region = spr.astype(np.int64) * lp + 16 * rng.integers(0, 2, n)
    rep_off = 32 + np.cumsum(region) - region
    total = (32 + int(region.sum()) + 64 + 31) // 32 * 32
    sh_off = (np.cumsum(L) - L).astype(np.uint64)
    sh = np.zeros((T, int(L.sum()) + 1), dtype=np.uint8)
    _data_shards_into(sh, arena, data_off, lens, d, sh_off)
    oracle.rs_encode_batch(d, p, arena, data_off, lens, sh[d:].reshape(-1), sh.shape[1], sh_off)
    canary = rng.integers(0, 256, (n_rep, total), dtype=np.uint8)
    want = canary.copy()
    for k in range(1, d + 1):                 # the reference's assignment, bit for bit
        asg = oracle.cw_brr_assignment(n_rep, T, k)
        for r in range(n_rep):
            assert int(asg[r]) == sum(1 << ((r * dj + kk) % T) for kk in range(k))
    for kk in range(d):
        sel = (spr > kk) & (lens > 0)
        dst = rep_off[sel] + kk * lp[sel]
        src = _ranges(sh_off[sel].astype(np.int64), L[sel])
        to = _ranges(dst, L[sel])
        zeros = _ranges(dst + L[sel], lp[sel] - L[sel])
        for r in range(n_rep):
            want[r, to] = sh[(r * dj + kk) % T, src]
            want[r, zeros] = 0
    B = _Dist()
    B.arena, B.data_off, B.lens, B.spr, B.rep_off, B.canary, B.want = arena, data_off, lens, spr, rep_off, canary, want
    return B


def _dist_dev(B):
    return (torch.from_numpy(B.arena).to(DEV), torch.from_numpy(B.data_off.astype(np.int64)).to(DEV),
            torch.from_numpy(B.lens.astype(np.int32)).to(DEV), torch.from_numpy(B.spr).to(DEV),
            torch.from_numpy(B.rep_off.astype(np.int64)).to(DEV))


def _distribute(rs, args, n, logs):
    import ctypes as C
    arr = (C.c_void_p * logs.shape[0])(*[logs[r].data_ptr() for r in range(logs.shape[0])])
    check(rs.lib.ss_crossword_distribute_dev(rs.h, *(a.data_ptr() for a in args), n, arr, logs.shape[0]))


# (n_replicas, d, p, variant, kernel, n values): the specialised RS(3,2) kernel, static and dynamic; the general kernel at
# every compile-time cluster code at a population dividing T, with run-time masks (bit 11, RS(3,2) through variant 4,
# codes without a table) and at populations 1, 8 and 16
def _dist_cases():
    st, gen = "crossword_distribute_generic_kernel<static>", "crossword_distribute_generic_kernel"
    return [
        (5, 3, 2, 0, "rs32_crossword_distribute_kernel<1>", "static"),
        (5, 3, 2, 6, "rs32_crossword_distribute_kernel<8,dynamic>", "dyn8"),
        (5, 3, 2, 7, "rs32_crossword_distribute_kernel<4,dynamic>", "dyn4"),
        (3, 2, 1, 0, st, "static"), (7, 4, 3, 0, st, "static"), (9, 5, 4, 0, st, "static"),
        (3, 4, 2, 0, st, "static"), (6, 4, 2, 0, st, "static"), (2, 3, 1, 0, st, "static"), (4, 3, 1, 0, st, "static"),
        (7, 4, 3, 1 << 11, gen, "static"), (5, 3, 2, 4, gen, "static"), (1, 3, 2, 0, gen, "static"),
        (8, 4, 4, 0, gen, "wrap"), (16, 8, 8, 0, gen, "wrap"),
    ]


DIST_CASES = _dist_cases()


def _dist_n_values(ctx, sched):
    cap = _ragged_cap(ctx)
    if sched == "static":
        return _grid_edges(cap)
    if sched == "wrap":                      # populations 8 and 16: one pass plus one codeword (host memory)
        return [cap + 1]
    run = 8 if sched == "dyn8" else 4
    dcap = ctx.sm_count * 3 * 8 * run       # codewords the dynamic grid takes in its first round of runs
    return [dcap - 1, dcap + 1, 3 * dcap + 5]


@pytest.mark.gpu
@pytest.mark.parametrize("n_rep,d,p,variant,kernel,sched", DIST_CASES)
def test_distribute_grid_edges(ctx, oracle, n_rep, d, p, variant, kernel, sched):
    rng = np.random.default_rng(800 + 10 * n_rep + d + variant)
    ns = _dist_n_values(ctx, sched)
    n_max = max(ns)
    if sched.startswith("dyn"):
        lens = _dyn_run_lengths(rng, n_max, 8 if sched == "dyn8" else 4)
        assert all(n % (8 if sched == "dyn8" else 4) for n in ns)
    else:
        lens = _short_lengths(rng, n_max, d)
    B = _dist_batch(oracle, d, p, n_rep, lens, 900 + n_rep + d)
    args = _dist_dev(B)
    rs = ReedSolomon(ctx, d, p)
    rs.set_variant(variant)
    canary = torch.from_numpy(B.canary).to(DEV)
    want = torch.from_numpy(B.want).to(DEV)
    for n in ns:
        logs = canary.clone()
        _distribute(rs, args, n, logs)
        torch.cuda.synchronize()
        assert rs.last_kernel() == kernel
        REACHED.add(kernel)
        cut = int(B.rep_off[n]) if n < n_max else logs.shape[1]
        _same(logs[:, :cut], want[:, :cut], f"n {n}: slots of the batch")
        _same(logs[:, cut:], canary[:, cut:], f"n {n}: logs past the batch")
    DONE.add(("dist", n_rep, d, p, variant))


@pytest.mark.gpu
@pytest.mark.parametrize("variant,kernel", [(6, "rs32_crossword_distribute_kernel<8,dynamic>"),
                                            (7, "rs32_crossword_distribute_kernel<4,dynamic>")])
def test_distribute_dynamic_back_to_back(ctx, oracle, variant, kernel):
    """two calls in a row on the stream, no synchronisation between them, different batches into different logs: each
    launch must start its counter of taken codewords from zero"""
    run = 8 if variant == 6 else 4
    dcap = ctx.sm_count * 3 * 8 * run
    rs = ReedSolomon(ctx, 3, 2)
    rs.set_variant(variant)
    rng = np.random.default_rng(1000 + variant)
    batches = [_dist_batch(oracle, 3, 2, 5, _dyn_run_lengths(rng, n, run), 1100 + variant + n)
               for n in (dcap + 3, 2 * dcap - 1)]
    devs = [_dist_dev(B) for B in batches]
    logs = [torch.from_numpy(B.canary).to(DEV) for B in batches]
    torch.cuda.synchronize()
    for B, a, lg in zip(batches, devs, logs):
        _distribute(rs, a, len(B.lens), lg)
        assert rs.last_kernel() == kernel
    torch.cuda.synchronize()
    REACHED.add(kernel)
    for i, (B, lg) in enumerate(zip(batches, logs)):
        _same(lg, torch.from_numpy(B.want).to(DEV), f"call {i}")
    DONE.add(("b2b", variant))


# ---------------------------------------------------------------------------------------------
# reach: every name the launchers can report was reached by the matrix above
# ---------------------------------------------------------------------------------------------
N_MATRIX = (2 * len(ROW_WIDTHS) + len(FALLBACK_CODES) + 1 + len(RAGGED_CASES) + len(DIST_CASES) + 2)


@pytest.mark.gpu
def test_every_reconstruct_and_distribute_kernel_reached():
    if len(DONE) != N_MATRIX:
        pytest.skip(f"{len(DONE)} of the {N_MATRIX} matrix cases ran; the reach check needs the whole file")
    assert REACHED == RECON_KERNELS | DIST_KERNELS
