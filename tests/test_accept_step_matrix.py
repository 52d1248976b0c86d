"""The fused accept step (ss_accept_step_fused_dev: encode a batch and tally each group's 64-slot ack window in one
launch) and the replicate step (ss_accept_step_replicate_dev, the EMIT instances of the same kernels) at every kernel
instance the launcher reaches, against two references each.

  * The tally is checked against a numpy restatement written here (count the set bits of every slot across the R planes,
    compare with the threshold, pack; commit_bar = the committed prefix, 64 for a full window), and the CPU oracle's
    tally must agree with that restatement, so a kernel and the oracle cannot drift together.
  * Parity is checked against oracle.rs_encode_uniform; with SS_RS_EMIT_DATA the data-shard planes against oracle.cw_split.

Every output lands in guarded buffers: sentinel bands around the shard planes and in each slot's slack past the written
length, guard words around committed / commit_bar, and all-ones poison words just before and after the R x n ack planes
(a kernel that reads the planes at the wrong stride or past their ends commits slots it should not).  Each case also pins
rs.last_kernel(), so it proves which instance ran.

Populations R in {1, 2, 3, 5, 7, 9, 15, 16} are not tied to d + p; thresholds cover 0, 1, a majority, R, R + 1, 31
(the five-bit counter's top), 32 and 2^32 - 1; ack densities are 0, 0.5, 0.9 and 1 with plane 0 (the leader's own ack)
all ones.  Group counts that depend on the grid are computed from the device's SM count with the launcher's formulas.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from summerset_b200 import workloads as wl
from summerset_b200._lib import check
from summerset_b200.api import ReedSolomon, round_up, shard_len

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PADDED16, EMIT_DATA = 1, 2          # SS_RS_OUT_PADDED16, SS_RS_EMIT_DATA
GUARD = 64                          # guard bytes around the shard planes; guard words around every other buffer
SENT = 0xC3                         # shard-plane sentinel
COM_SENT = 0x5A5A5A5A5A5A5A5A
BAR_SENT = 0x3C3C3C3C
ALL = np.uint64(0xFFFFFFFFFFFFFFFF)
BULK = 1 << 18

# (R, threshold, ack density): every population, every threshold edge, every density.  Each fused case runs all of them.
TALLIES = [
    (1, 0, 0.0), (1, 1, 0.0), (1, 2, 1.0),
    (2, 2, 0.5), (2, 1, 0.9),
    (3, 2, 0.9), (3, 4, 1.0),
    (5, 3, 0.5), (5, 5, 0.9), (5, 4, 1.0),
    (7, 4, 0.9), (7, 8, 1.0),
    (9, 5, 0.5), (9, 9, 1.0),
    (15, 8, 0.9), (15, 31, 1.0), (15, 15, 1.0),
    (16, 9, 0.9), (16, 16, 1.0), (16, 17, 1.0), (16, 1, 0.0),
    (16, 31, 1.0), (16, 32, 1.0), (16, 2 ** 32 - 1, 1.0),
]
# a short list for the large grid-edge batches: a majority at R = 5, a full window, the 16-plane counter
TALLIES_SHORT = [(5, 3, 0.5), (3, 2, 1.0), (16, 16, 0.9)]


# ---------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------
def ref_tally(planes, threshold):
    """planes uint64 [R, n] -> (committed uint64 [n], commit_bar uint32 [n]): per group and slot, count the acks across
    the R planes and commit the slot when the count reaches the threshold; commit_bar is the committed prefix."""
    R, n = planes.shape
    bits = np.unpackbits(np.ascontiguousarray(planes).view(np.uint8).reshape(R, n, 8), axis=2, bitorder="little")
    ok = bits.sum(axis=0, dtype=np.int64) >= threshold                          # [n, 64]
    committed = np.packbits(ok, axis=1, bitorder="little").view("<u8").reshape(n)
    bar = np.where(ok.all(axis=1), 64, np.argmin(ok, axis=1)).astype(np.uint32)
    return committed, bar


def ack_planes(R, n, density, seed):
    """R ack planes for n groups: plane 0 is the leader's own ack (all ones), the others set each slot with `density`."""
    rng = np.random.default_rng(seed)
    planes = np.zeros((R, n), dtype=np.uint64)
    planes[0] = ALL
    for r in range(1, R):
        if density >= 1.0:
            planes[r] = ALL
        elif density > 0.0:
            bits = rng.random((n, 64)) < density
            planes[r] = np.packbits(bits, axis=1, bitorder="little").view("<u8").reshape(n)
    return planes


def data_shards(data, data_len, d):
    """the d data shards of every codeword, zero-padded to L: uint8 [d, n, L]"""
    n = data.shape[0]
    L = shard_len(data_len, d)
    flat = np.zeros((n, d * L), dtype=np.uint8)
    flat[:, :data_len] = data[:, :data_len]
    return flat.reshape(n, d, L).transpose(1, 0, 2)


def horner_kernel(d, data_len, tag):
    """The Horner kernel the row geometry takes: packed when the one-codeword-per-pass layout would idle or mask lanes
    and the codeword fits 256 columns, else the row kernel."""
    L = shard_len(data_len, d)
    vpc = -(-L // 16)
    fc = min(L, max(0, data_len - (d - 1) * L)) // 16
    row_threads = 256 if vpc > 256 else round_up(vpc, 32)
    packed = (fc != vpc or row_threads != vpc) and vpc <= 256
    return ("horner_encode_packed_kernel" if packed else "horner_encode_row_kernel") + tag + "+tally"


@pytest.fixture(scope="module")
def coder(ctx):
    """one coder per code for the whole file"""
    made = {}

    def get(d, p):
        if (d, p) not in made:
            made[(d, p)] = ReedSolomon(ctx, d, p)
        return made[(d, p)]

    yield get
    for rs in made.values():
        rs.close()


# ---------------------------------------------------------------------------------------------
# the harness
# ---------------------------------------------------------------------------------------------
class Batch:
    """One batch of payloads on the device (optionally at a misaligned base) and its expected parity / data shards."""

    def __init__(self, oracle, d, p, data_len, n, stride=None, misalign=0, seed=0):
        self.d, self.p, self.data_len, self.n = d, p, data_len, n
        self.stride = stride if stride is not None else round_up(max(data_len, 1), 16)
        self.data = wl.payload_uniform(n, data_len, stride=self.stride, seed_extra=seed * 7919 + data_len + n)
        self.buf = torch.full((misalign + n * self.stride + 64,), 0xA5, dtype=torch.uint8, device=DEV)
        self.buf[misalign:misalign + n * self.stride] = torch.from_numpy(self.data.reshape(-1)).to(DEV)
        self.ptr = self.buf.data_ptr() + misalign
        self.L = shard_len(data_len, d) if data_len else 0
        self.parity = oracle.rs_encode_uniform(d, p, self.data, data_len) if data_len else None
        self.shards = data_shards(self.data, data_len, d) if data_len else None
        if data_len:
            # the oracle's codeword split agrees with the vectorised one used below (sampled codewords)
            for g in sorted({0, n // 2, n - 1}):
                assert (oracle.cw_split(self.data[g, :data_len].tobytes(), d) == self.shards[:, g]).all()


def _guarded(n_words, fill, dtype):
    return torch.full((n_words + 2 * GUARD,), fill, dtype=dtype, device=DEV)


def _tally_buffers(planes, with_bar):
    R, n = planes.shape
    ack = _guarded(R * n, -1, torch.int64)                           # all-ones poison words before and after the planes
    ack[GUARD:GUARD + R * n] = torch.from_numpy(planes.reshape(-1).view(np.int64)).to(DEV)
    com = _guarded(n, COM_SENT, torch.int64)
    bar = _guarded(n, BAR_SENT, torch.int32)
    bar_ptr = bar.data_ptr() + 4 * GUARD if with_bar else None
    return ack, com, bar, ack.data_ptr() + 8 * GUARD, com.data_ptr() + 8 * GUARD, bar_ptr


def _check_tally(oracle, planes, threshold, com, bar, with_bar, what):
    n = planes.shape[1]
    want_c, want_b = ref_tally(planes, threshold)
    oc, ob = oracle.tally_planes(planes, threshold)
    assert (oc == want_c).all() and (ob == want_b).all(), f"{what}: the oracle's tally disagrees with the restatement"
    com = com.cpu().numpy().view(np.uint64)
    bar = bar.cpu().numpy().view(np.uint32)
    assert (com[:GUARD] == COM_SENT).all() and (com[GUARD + n:] == COM_SENT).all(), f"{what}: guard words of committed written"
    got = com[GUARD:GUARD + n]
    bad = np.flatnonzero(got != want_c)
    assert bad.size == 0, f"{what}: committed differs at {bad.size} groups, first {bad[:8]}"
    if with_bar:
        assert (bar[:GUARD] == BAR_SENT).all() and (bar[GUARD + n:] == BAR_SENT).all(), f"{what}: guard words of commit_bar written"
        bad = np.flatnonzero(bar[GUARD:GUARD + n] != want_b)
        assert bad.size == 0, f"{what}: commit_bar differs at {bad.size} groups, first {bad[:8]}"
    else:
        assert (bar == BAR_SENT).all(), f"{what}: commit_bar written although it was NULL"


def _check_planes(batch, out, ss, padded, emit, what):
    """the d + p shard planes: guard bands, slack past the written length of every slot, parity byte for byte, and the
    data-shard planes either equal to the oracle's split (SS_RS_EMIT_DATA) or untouched"""
    n, d, p, L = batch.n, batch.d, batch.p, batch.L
    nplanes = d + p
    body_len = nplanes * n * ss
    out = out.cpu().numpy()
    assert (out[:GUARD] == SENT).all() and (out[GUARD + body_len:] == SENT).all(), f"{what}: guard band around the planes written"
    body = out[GUARD:GUARD + body_len].reshape(nplanes, n, ss)
    vb = round_up(L, 16) if padded else L                            # bytes a slot receives
    assert (body[:, :, vb:] == SENT).all(), f"{what}: slack of a shard slot written"
    if not emit:
        assert (body[:d] == SENT).all(), f"{what}: data-shard planes written without SS_RS_EMIT_DATA"
    if batch.data_len == 0:
        return
    par = body[nplanes - p:]
    assert (par[:, :, :L] == batch.parity[:, :, :L]).all(), f"{what}: parity differs from the oracle"
    assert (par[:, :, L:vb] == 0).all(), f"{what}: padding of a parity slot is not zero"
    if emit:
        assert (body[:d, :, :L] == batch.shards).all(), f"{what}: data shards differ from the oracle's split"
        assert (body[:d, :, L:vb] == 0).all(), f"{what}: padding of a data-shard slot is not zero"


def fused(ctx, oracle, rs, batch, kernel, variant=0, flags=PADDED16, ss_extra=16, tallies=TALLIES, seed=0):
    """Runs the fused accept step on `batch` once per (R, threshold, density) in `tallies` and checks every output."""
    d, p, n = batch.d, batch.p, batch.n
    padded = bool(flags & PADDED16)
    emit = bool(flags & EMIT_DATA)
    vb = round_up(batch.L, 16) if padded else batch.L
    ss = vb + ss_extra
    for i, (R, thr, density) in enumerate(tallies):
        with_bar = i % 4 != 3
        what = f"({d},{p}) len {batch.data_len} n {n} variant {variant:#x} flags {flags} R {R} threshold {thr} density {density}"
        planes = ack_planes(R, n, density, seed=seed * 131 + i)
        # d + p planes in every case, parity at plane d: without SS_RS_EMIT_DATA the data-shard planes in front of the
        # parity are a sentinel region the kernel must not write
        out = torch.full((2 * GUARD + (d + p) * n * ss,), SENT, dtype=torch.uint8, device=DEV)
        base = out.data_ptr() + GUARD
        ack, com, bar, ack_ptr, com_ptr, bar_ptr = _tally_buffers(planes, with_bar)
        rs.set_variant(variant)
        try:
            check(ctx.lib.ss_accept_step_fused_dev(rs.h, batch.ptr, batch.stride, batch.data_len, n,
                                                   base + d * n * ss, n * ss, ss, flags,
                                                   ack_ptr, R, thr, com_ptr, bar_ptr))
            torch.cuda.synchronize()
        finally:
            rs.set_variant(0)
        assert rs.last_kernel() == kernel, what
        _check_tally(oracle, planes, thr, com, bar, with_bar, what)
        _check_planes(batch, out, ss, padded, emit, what)


# ---------------------------------------------------------------------------------------------
# the matrix: each case reaches a distinct instance or edge
# ---------------------------------------------------------------------------------------------
ROW = "rs32_encode_row_kernel+tally"
EMIT_ROW = "rs32_encode_row_kernel+tally"        # the EMIT instances report the row kernel's name
SEG = "rs32_encode_row_kernel<segmented>+tally"
BULK_K = "rs32_accept_bulk_kernel+tally"
FLAT32 = "rs32_encode_uniform_kernel+tally"
HFLAT = "horner_encode_uniform_kernel"          # the flat Horner and bit-plane kernels tally without saying so
GFLAT = "generic_encode_uniform_kernel"

# RS(3,2): (id, data_len, n, variant, flags, data stride (None: round_up(len, 16)), misaligned base, kernel)
RS32_CASES = [
    # the row kernel at the column edges (<false,128,12,PF>; 12288 is 256 columns: <false,256,4>)
    *[(f"row-len{L}", L, 37, 0, PADDED16, None, 0, ROW) for L in (1, 15, 16, 17, 4095, 4096, 4097, 12288)],
    ("row-n1", 4096, 1, 0, PADDED16, None, 0, ROW),
    ("row-n2", 17, 2, 0, PADDED16, None, 0, ROW),
    ("row-stride+16", 4095, 37, 0, PADDED16, 4096 + 16, 0, ROW),
    # register budgets (bits 0-3: 3 = 32 regs, 6 = 64, 7 = 56; 2 keeps the default instance)
    *[(f"row-budget{v}", 4096, 37, v, PADDED16, None, 0, ROW) for v in (2, 3, 6, 7)],
    ("row-budget7-len17", 17, 37, 7, PADDED16, None, 0, ROW),
    # chunked CTAs, every wave count, store cache modes, the fixed warp -> block assignment.  At n = 37 the launcher caps
    # the grid at n, so these cases pin each knob's kernel instance and its bytes on a CTA-per-codeword grid only; the
    # schedules themselves (waves, chunks, warp rotation) are exercised by test_grid_edges and test_multi_warp_ctas_stride
    ("row-chunked", 4096, 37, 1 << 4, PADDED16, None, 0, ROW),
    *[(f"row-waves{w}", 4096, 37, w << 5, PADDED16, None, 0, ROW) for w in range(1, 8)],
    *[(f"row-store{m}", 4096, 37, m << 8, PADDED16, None, 0, ROW) for m in (1, 2, 3)],
    ("row-fixed-warps", 4096, 37, 1 << 10, PADDED16, None, 0, ROW),
    ("row-fixed-warps-256", 12288, 37, 1 << 10, PADDED16, None, 0, ROW),
    ("row-chunked-1wave-fixed", 4097, 37, (1 << 4) | (1 << 5) | (1 << 10), PADDED16, None, 0, ROW),
    ("row-variant5", 4096, 37, 5, PADDED16, None, 0, ROW),            # bit-plane selector: RS(3,2) keeps its row kernel
    # the segmented row kernel (more than 256 columns)
    ("segmented", 12289, 37, 0, PADDED16, None, 0, SEG),
    ("segmented-store3", 12289, 5, 3 << 8, PADDED16, None, 0, SEG),
    # the bulk-copy kernel
    *[(f"bulk-len{L}", L, 37, BULK, PADDED16, None, 0, BULK_K) for L in (1, 17, 4096, 12288)],
    ("bulk-n1", 4096, 1, BULK, PADDED16, None, 0, BULK_K),
    ("bulk-interleave", 4095, 37, BULK | (1 << 21) | (3 << 19), PADDED16, None, 0, BULK_K),
    # the flat kernel: variant 1, byte-exact layout, odd stride, misaligned base, the tally alone
    ("flat-variant1", 4096, 37, 1, PADDED16, None, 0, FLAT32),
    ("flat-exact", 4097, 37, 0, 0, None, 0, FLAT32),
    ("flat-odd-stride", 4100, 37, 0, PADDED16, 4101, 0, FLAT32),
    ("flat-misaligned", 4096, 37, 0, PADDED16, None, 1, FLAT32),
    ("flat-len0", 0, 37, 0, PADDED16, None, 0, FLAT32),
    ("flat-len0-n1", 0, 1, 0, PADDED16, None, 0, FLAT32),
    ("flat-emit", 4097, 37, 1, PADDED16 | EMIT_DATA, None, 0, FLAT32),
    # SS_RS_EMIT_DATA: the EMIT instances (tally first, 64 waves)
    *[(f"emit-len{L}", L, 37, 0, PADDED16 | EMIT_DATA, None, 0, EMIT_ROW) for L in (17, 4096, 12288)],
    ("emit-store2", 4096, 37, 2 << 8, PADDED16 | EMIT_DATA, None, 0, EMIT_ROW),
    ("emit-segmented", 12289, 5, 0, PADDED16 | EMIT_DATA, None, 0, SEG),
    ("emit-bulk-bit", 4096, 37, BULK, PADDED16 | EMIT_DATA, None, 0, EMIT_ROW),   # the bulk kernel has no EMIT form
]


@pytest.mark.parametrize("name,data_len,n,variant,flags,stride,misalign,kernel", RS32_CASES, ids=[c[0] for c in RS32_CASES])
def test_rs32(ctx, oracle, coder, name, data_len, n, variant, flags, stride, misalign, kernel):
    batch = Batch(oracle, 3, 2, data_len, n, stride=stride, misalign=misalign, seed=len(name))
    fused(ctx, oracle, coder(3, 2), batch, kernel, variant=variant, flags=flags, ss_extra=16 if flags & PADDED16 else 3)


STATIC = [(2, 1), (3, 1), (4, 2), (4, 3), (5, 4)]


def _horner_cases():
    cases = []
    for d, p in STATIC:
        row = d * 512                                      # L = 512: 32 complete columns, the row kernel
        cases.append((f"{d}{p}-row", d, p, row, 37, 0, PADDED16))
        cases.append((f"{d}{p}-packed", d, p, 4095, 37, 0, PADDED16))
        for v in (2, 3, 4):                                # register budgets of the row kernel
            cases.append((f"{d}{p}-row-budget{v}", d, p, row, 37, v, PADDED16))
    # the column edges on the 7-replica code, and the 256-thread and wider-than-a-CTA row kernels
    for L in (1, 15, 16, 17, 4096, 4097, 12288, 12289):
        cases.append((f"43-len{L}", 4, 3, L, 23, 0, PADDED16))
    cases.append(("21-len12289", 2, 1, 12289, 11, 0, PADDED16))
    cases.append(("43-n1", 4, 3, 4096, 1, 0, PADDED16))
    cases.append(("43-n2", 4, 3, 4095, 2, 0, PADDED16))
    # forced layouts (bit 13 off, bit 14 on) and the pipelined packed loop (bit 15)
    cases.append(("43-force-row", 4, 3, 4095, 37, 1 << 13, PADDED16))
    cases.append(("43-force-packed", 4, 3, 2048, 37, 1 << 14, PADDED16))
    cases.append(("43-packed-pipe", 4, 3, 4090, 37, (1 << 14) | (1 << 15), PADDED16))   # L = 1023: unaligned shards
    # the coder's NVRTC specialisation, then run-time masks (bit 11) and NVRTC skipped (bit 17)
    for v, tag in ((0, "nvrtc"), (1 << 11, "masks"), (1 << 17, "no-nvrtc")):
        cases.append((f"64-row-{tag}", 6, 4, 6 * 512, 37, v, PADDED16))
        cases.append((f"64-packed-{tag}", 6, 4, 4090, 37, v, PADDED16))
    cases.append(("64-row-masks-budget4", 6, 4, 6 * 512, 37, (1 << 11) | 4, PADDED16))
    cases.append(("43-masks-budget3", 4, 3, 2048, 37, (1 << 11) | 3, PADDED16))
    # SS_RS_EMIT_DATA
    cases.append(("43-emit-row", 4, 3, 4096, 37, 0, PADDED16 | EMIT_DATA))
    cases.append(("54-emit-packed", 5, 4, 4095, 37, 0, PADDED16 | EMIT_DATA))
    cases.append(("64-emit-nvrtc", 6, 4, 4090, 37, 0, PADDED16 | EMIT_DATA))
    return cases


HORNER_CASES = _horner_cases()


def _horner_expected(d, p, data_len, variant):
    static = (d, p) in STATIC
    masks = (variant >> 11) & 1
    tag = "" if masks else "<static code>" if static else "" if (variant >> 17) & 1 else "<nvrtc>"
    name = horner_kernel(d, data_len, tag)
    if (variant >> 13) & 1:
        name = name.replace("packed", "row")
    if (variant >> 14) & 1:
        name = name.replace("_row_", "_packed_")
    return name


@pytest.mark.parametrize("name,d,p,data_len,n,variant,flags", HORNER_CASES, ids=[c[0] for c in HORNER_CASES])
def test_horner(ctx, oracle, coder, name, d, p, data_len, n, variant, flags):
    batch = Batch(oracle, d, p, data_len, n, seed=d * 16 + p)
    fused(ctx, oracle, coder(d, p), batch, _horner_expected(d, p, data_len, variant), variant=variant, flags=flags)


# flat Horner and bit-plane kernels: (id, d, p, data_len, n, variant, flags, stride, misalign, kernel)
FLAT_CASES = [
    ("43-variant1", 4, 3, 4096, 37, 1, PADDED16, None, 0, HFLAT),
    ("54-exact", 5, 4, 4097, 37, 0, 0, None, 0, HFLAT),
    ("21-exact-len1", 2, 1, 1, 37, 0, 0, None, 0, HFLAT),
    ("43-odd-stride", 4, 3, 1000, 37, 0, PADDED16, 1003, 0, HFLAT),
    ("64-misaligned", 6, 4, 4090, 37, 0, PADDED16, None, 5, HFLAT),
    ("43-len0", 4, 3, 0, 37, 0, PADDED16, None, 0, HFLAT),
    ("43-variant1-emit", 4, 3, 4095, 37, 1, PADDED16 | EMIT_DATA, None, 0, HFLAT),
    ("42-variant5", 4, 2, 4096, 37, 5, PADDED16, None, 0, GFLAT),
    ("43-variant5-exact", 4, 3, 17, 37, 5, 0, None, 0, GFLAT),
    ("96", 9, 6, 4096, 37, 0, PADDED16, None, 0, GFLAT),
    ("96-len17", 9, 6, 17, 37, 0, PADDED16, None, 0, GFLAT),
    ("128-exact", 12, 8, 12289, 11, 0, 0, None, 0, GFLAT),
    ("128-emit", 12, 8, 4097, 11, 0, PADDED16 | EMIT_DATA, None, 0, GFLAT),
    ("96-len0", 9, 6, 0, 37, 0, PADDED16, None, 0, GFLAT),
]


@pytest.mark.parametrize("name,d,p,data_len,n,variant,flags,stride,misalign,kernel", FLAT_CASES,
                         ids=[c[0] for c in FLAT_CASES])
def test_flat(ctx, oracle, coder, name, d, p, data_len, n, variant, flags, stride, misalign, kernel):
    batch = Batch(oracle, d, p, data_len, n, stride=stride, misalign=misalign, seed=d * 16 + p + 1)
    fused(ctx, oracle, coder(d, p), batch, kernel, variant=variant, flags=flags, ss_extra=16 if flags & PADDED16 else 3)


# ---------------------------------------------------------------------------------------------
# grid edges: group counts just below, at and above each schedule's CTA count (computed as encode_rs32_row does)
#
# Not reached here: the CTA caps of the Horner row kernel (64 waves of CTAs, at least 270k codewords of >= 512-byte shards)
# and of the packed kernel's main grid.  Their per-CTA tally slices are exercised only with grid = n (row) or the small
# tail + main grid of a short batch (packed); test_gpu_rs.py's 400,000-group fused step wraps the Horner row grid.
# ---------------------------------------------------------------------------------------------
GRID_LEN = 48                      # L = 16: one column, 32-thread CTAs, 32 resident per SM


def _row_grid(sm, waves):
    per_sm = min(32, 2048 // 32)
    return sm * per_sm * waves


SCHEDULES = {
    # name: (variant, CTA count for GRID_LEN payloads, kernel)
    "1wave": (1 << 5, lambda sm: _row_grid(sm, 1), ROW),
    "4waves": (3 << 5, lambda sm: _row_grid(sm, 4), ROW),
    "1wave-chunked": ((1 << 4) | (1 << 5), lambda sm: _row_grid(sm, 1), ROW),
    "1wave-fixed-warps": ((1 << 5) | (1 << 10), lambda sm: _row_grid(sm, 1), ROW),
    "bulk": (BULK, lambda sm: sm * 4, BULK_K),           # 4 resident CTAs per SM (bits 19-20 = 0)
}
WHERE = {"below": lambda g: g - 1, "at": lambda g: g, "above": lambda g: g + 1, "ragged": lambda g: 2 * g + g // 3 + 1,
         "wrap": lambda g: 3 * g + 77}


@pytest.mark.parametrize("where", list(WHERE))
@pytest.mark.parametrize("schedule", list(SCHEDULES))
def test_grid_edges(ctx, oracle, coder, schedule, where):
    """n around the CTA count: the last tally slice short or empty, CTAs that stride over several codewords"""
    variant, grid, kernel = SCHEDULES[schedule]
    n = WHERE[where](grid(ctx.sm_count))
    batch = Batch(oracle, 3, 2, GRID_LEN, n, seed=n)
    fused(ctx, oracle, coder(3, 2), batch, kernel, variant=variant, tallies=TALLIES_SHORT, seed=n)


@pytest.mark.parametrize("where", ["below", "at", "above"])
def test_emit_grid_edges(ctx, oracle, coder, where):
    """SS_RS_EMIT_DATA keeps 64 waves of CTAs and tallies before the encode loop: n around that grid"""
    n = WHERE[where](_row_grid(ctx.sm_count, 64))
    batch = Batch(oracle, 3, 2, GRID_LEN, n, seed=n)
    fused(ctx, oracle, coder(3, 2), batch, EMIT_ROW, flags=PADDED16 | EMIT_DATA, tallies=TALLIES_SHORT[:2], seed=n)


ROT_LEN = 4096                     # L = 1366: 86 columns, 96-thread CTAs (three warps, the last block masked), 21 per SM


@pytest.mark.parametrize("schedule", ["rotating", "fixed-warps", "chunked", "emit-rotating", "emit-fixed-warps"])
def test_multi_warp_ctas_stride(ctx, oracle, coder, schedule):
    """A single wave of three-warp CTAs over n = 3 * grid + 77 codewords: every CTA encodes four or more codewords, so
    the warp -> column-block assignment (rotating by default, fixed with bit 10) decides which warp writes which block
    of each codeword -- a rotation that skips or repeats a block leaves columns unwritten"""
    grid = ctx.sm_count * (2048 // 96)
    n = 3 * grid + 77
    emit = schedule.startswith("emit")
    variant = (1 << 5) | ((1 << 10) if "fixed" in schedule else 0) | ((1 << 4) if schedule == "chunked" else 0)
    batch = Batch(oracle, 3, 2, ROT_LEN, n, seed=n + len(schedule))
    fused(ctx, oracle, coder(3, 2), batch, EMIT_ROW if emit else ROW, variant=variant,
          flags=PADDED16 | (EMIT_DATA if emit else 0), tallies=TALLIES_SHORT[:2], seed=n)


def test_default_row_schedule_large_batch(ctx, oracle, coder):
    """the default schedule (a CTA per codeword) past 65535 CTAs, where the tally slice of every CTA is one group"""
    n = 70001
    batch = Batch(oracle, 3, 2, GRID_LEN, n, seed=3)
    fused(ctx, oracle, coder(3, 2), batch, ROW, tallies=TALLIES_SHORT[:1])


# ---------------------------------------------------------------------------------------------
# regression guards for the tally word itself, on the hot kernel
# ---------------------------------------------------------------------------------------------
def test_sixteen_acks_need_the_fifth_counter_bit(ctx, oracle, coder):
    """16 acks on every slot: a four-bit counter wraps to 0 and commits nothing at thresholds 9..16"""
    batch = Batch(oracle, 3, 2, 4096, 19, seed=16)
    fused(ctx, oracle, coder(3, 2), batch, ROW, tallies=[(16, t, 1.0) for t in (1, 9, 15, 16, 17)])


def test_thresholds_past_the_counter(ctx, oracle, coder):
    """thresholds 32 .. 2^32 - 1 commit nothing even with every ack in; 31 is the counter's largest comparable value"""
    batch = Batch(oracle, 3, 2, 4096, 19, seed=32)
    fused(ctx, oracle, coder(3, 2), batch, ROW,
          tallies=[(16, t, 1.0) for t in (31, 32, 33, 63, 64, 1 << 16, 2 ** 31, 2 ** 32 - 1)])


def test_full_window_commit_bar_is_64(ctx, oracle, coder):
    """a window committed in every slot has commit_bar 64 on every kernel family"""
    full = [(5, 4, 1.0), (1, 1, 0.0), (16, 0, 0.0)]
    for d, p, data_len, variant, kernel in ((3, 2, 4096, 0, ROW), (3, 2, 4096, BULK, BULK_K), (3, 2, 4096, 1, FLAT32),
                                            (4, 3, 4095, 0, "horner_encode_packed_kernel<static code>+tally"),
                                            (4, 3, 2048, 0, "horner_encode_row_kernel<static code>+tally"),
                                            (9, 6, 100, 0, GFLAT), (4, 3, 100, 1, HFLAT)):
        batch = Batch(oracle, d, p, data_len, 9, seed=64)
        fused(ctx, oracle, coder(d, p), batch, kernel, variant=variant, tallies=full)


# ---------------------------------------------------------------------------------------------
# the replicate step on one GPU: every shard plane a separate local buffer
# ---------------------------------------------------------------------------------------------
REPLICATE_CASES = [
    ("32-row", 3, 2, 4096, 37, 0, EMIT_ROW),
    ("32-row-len17", 3, 2, 17, 37, 0, EMIT_ROW),
    ("32-row-256", 3, 2, 12288, 13, 0, EMIT_ROW),
    ("32-segmented", 3, 2, 12289, 5, 0, SEG),
    ("32-variant1", 3, 2, 4096, 37, 1, EMIT_ROW),           # the flat selector is ignored: no peer-plane mode there
    ("43-row", 4, 3, 4096, 37, 0, "horner_encode_row_kernel<static code>+tally"),
    ("54-packed", 5, 4, 4095, 37, 5, "horner_encode_packed_kernel<static code>+tally"),
    ("64-nvrtc", 6, 4, 4090, 37, 0, "horner_encode_packed_kernel<nvrtc>+tally"),
]


@pytest.mark.parametrize("name,d,p,data_len,n,variant,kernel", REPLICATE_CASES, ids=[c[0] for c in REPLICATE_CASES])
def test_replicate(ctx, oracle, coder, name, d, p, data_len, n, variant, kernel):
    rs = coder(d, p)
    batch = Batch(oracle, d, p, data_len, n, seed=d + p + 100)
    L = batch.L
    vb = round_up(L, 16)
    ss = vb + 16
    for i, (R, thr, density) in enumerate(TALLIES):
        with_bar = i % 4 != 3
        what = f"replicate ({d},{p}) len {data_len} R {R} threshold {thr} density {density}"
        planes = ack_planes(R, n, density, seed=1000 + i)
        outs = [torch.full((2 * GUARD + n * ss,), SENT, dtype=torch.uint8, device=DEV) for _ in range(d + p)]
        ptrs = (C.c_void_p * (d + p))(*[o.data_ptr() + GUARD for o in outs])
        ack, com, bar, ack_ptr, com_ptr, bar_ptr = _tally_buffers(planes, with_bar)
        rs.set_variant(variant)
        try:
            check(ctx.lib.ss_accept_step_replicate_dev(rs.h, batch.ptr, batch.stride, data_len, n, ptrs, ss,
                                                       ack_ptr, R, thr, com_ptr, bar_ptr, None))
            torch.cuda.synchronize()
        finally:
            rs.set_variant(0)
        assert rs.last_kernel() == kernel, what
        _check_tally(oracle, planes, thr, com, bar, with_bar, what)
        for j, o in enumerate(outs):
            o = o.cpu().numpy()
            assert (o[:GUARD] == SENT).all() and (o[GUARD + n * ss:] == SENT).all(), f"{what}: guard band of plane {j} written"
            slot = o[GUARD:GUARD + n * ss].reshape(n, ss)
            assert (slot[:, vb:] == SENT).all(), f"{what}: slack of plane {j} written"
            want = batch.shards[j] if j < d else batch.parity[j - d, :, :L]
            assert (slot[:, :L] == want).all(), f"{what}: shard plane {j} differs from the oracle"
            assert (slot[:, L:vb] == 0).all(), f"{what}: padding of plane {j} is not zero"


# ---------------------------------------------------------------------------------------------
# the restatement itself, on hand-made windows (runs with the rest of the file)
# ---------------------------------------------------------------------------------------------
def test_reference_tally_on_known_windows(oracle):
    planes = np.array([[ALL, 0, 1, ALL], [ALL, 0, 3, ALL ^ np.uint64(1 << 40)], [0, 0, 7, ALL]], dtype=np.uint64)
    c, b = ref_tally(planes, 2)
    assert c.tolist() == [int(ALL), 0, 3, int(ALL)] and b.tolist() == [64, 0, 2, 64]
    c, b = ref_tally(planes, 3)
    assert c.tolist() == [0, 0, 1, int(ALL) ^ (1 << 40)] and b.tolist() == [0, 0, 1, 40]
    for thr in (0, 1, 2, 3, 4, 31, 32, 2 ** 32 - 1):
        oc, ob = oracle.tally_planes(planes, thr)
        c, b = ref_tally(planes, thr)
        assert (oc == c).all() and (ob == b).all(), thr
