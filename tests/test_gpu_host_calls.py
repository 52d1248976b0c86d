"""The host-memory Reed-Solomon entry points against the CPU oracle: the crate-shaped single-codeword calls
(ss_rs_encode / ss_rs_reconstruct / ss_rs_reconstruct_data / ss_rs_verify, what a Summerset build's RSCodeword links
against) and the chunked host-buffer batch calls (ss_rs_encode_uniform / ss_accept_step_fused).

Every call goes through the raw C ABI so the test controls the memory it hands over: shards are separate slices at odd
addresses with canary bytes between them, missing parity entries of reconstruct_data alias one shared buffer, and
host batch buffers end exactly at the last payload.  Each case checks the result byte for byte against the oracle
(oracle/ss_oracle.c) and checks that no byte outside the slots the call defines changed."""
import ctypes as C
import functools
import threading

import numpy as np
import pytest
import torch

from summerset_b200 import _lib
from summerset_b200.api import Context, ReedSolomon, round_up, shard_len

pytestmark = pytest.mark.gpu

STAGED_CALL_LIMIT = 8 << 20        # capi.cu kStagedCallLimit: larger single codewords copy straight from the slices
CANARY, GARBAGE = 0xA5, 0xCC
STATIC_CODES = {(2, 1), (3, 1), (4, 2), (4, 3), (5, 4)}   # static_codes.hpp; (3,2) has kernels of its own


@pytest.fixture(scope="module")
def coder(ctx):
    """one coder per code for the whole file: NVRTC specialises each code's kernel once"""
    cache = {}

    def get(d, p):
        if (d, p) not in cache:
            cache[(d, p)] = ReedSolomon(ctx, d, p)
        return cache[(d, p)]
    yield get
    for rs in cache.values():
        rs.close()


def _ptrs(bufs):
    return (C.c_void_p * len(bufs))(*[b.ctypes.data for b in bufs])


def _err():
    return _lib.load().ss_last_error().decode()


# ---------------------------------------------------------------------------------------------------------------------
# memory layouts
# ---------------------------------------------------------------------------------------------------------------------
def _data_slices(d, L, rng):
    """d random shards inside one canary-filled buffer, each starting at an odd address with a gap after it"""
    pitch = L + 1 if L % 2 else L + 2                 # even pitch: every slice starts at an odd offset
    buf = np.full(2 + d * pitch, CANARY, dtype=np.uint8)
    sl = [buf[1 + i * pitch:1 + i * pitch + L] for i in range(d)]
    for s in sl:
        s[:] = rng.integers(0, 256, L, dtype=np.uint8)
    assert all(s.ctypes.data % 2 == 1 for s in sl)
    return buf, sl


def _parity_slices(p, L, fill=CANARY):
    """p views into one canary buffer with 1-15 canary bytes before, between and after them"""
    gaps = [1 + (7 * j + L) % 15 for j in range(p + 1)]
    offs, pos = [], gaps[0]
    for j in range(p):
        offs.append(pos)
        pos += L + gaps[j + 1]
    buf = np.full(pos, CANARY, dtype=np.uint8)
    sl = [buf[o:o + L] for o in offs]
    for s in sl:
        s[:] = fill
    return buf, sl, offs


def _oracle_parity(oracle, d, p, data):
    L = len(data[0])
    shards = [s.copy() for s in data] + [np.zeros(L, dtype=np.uint8) for _ in range(p)]
    assert oracle.rs_encode(d, p, shards) == 0
    return shards[d:]


def _codeword(oracle, d, p, L, seed):
    """an oracle-encoded codeword [d+p, L]"""
    rng = np.random.default_rng(seed)
    data = [rng.integers(0, 256, L, dtype=np.uint8) for _ in range(d)]
    return np.stack(data + _oracle_parity(oracle, d, p, data))


def _oracle_reconstruct(oracle, d, p, bufs, present, data_only):
    """ssor_rs_reconstruct in place on bufs; -> (rc, present after the call)"""
    pres = np.ascontiguousarray(present, dtype=np.uint8).copy()
    rc = oracle.lib().ssor_rs_reconstruct(d, p, _ptrs(bufs), pres.ctypes.data_as(C.c_void_p), C.c_size_t(len(bufs[0])),
                                          1 if data_only else 0)
    return int(rc), pres


# ---------------------------------------------------------------------------------------------------------------------
# A. ss_rs_encode: every code class x every shard-length class
# ---------------------------------------------------------------------------------------------------------------------
def predict_encode_kernel(d, p, L):
    """the kernel launch_rs_encode picks for ss_rs_encode's batch of one (rs_kernels.cu): payload stride d*L, padded
    shard slots of round_up(L,16), a 256-byte aligned device payload, default variant"""
    vpc = -(-L // 16)
    row = (d * L) % 16 == 0                          # 16-byte payload rows: the row kernels take it
    if (d, p) == (3, 2):
        if not row:
            return "rs32_encode_uniform_kernel"
        return "rs32_encode_row_kernel<segmented>" if vpc > 256 else "rs32_encode_row_kernel"
    if d > 8:
        return "generic_encode_uniform_kernel"
    if not row:
        return "horner_encode_uniform_kernel"
    fast_cols = L // 16                              # the last shard lies wholly in the payload
    row_threads = 256 if vpc > 256 else round_up(vpc, 32)
    packed = (fast_cols != vpc or row_threads != vpc) and vpc <= 256
    tag = "<static code>" if (d, p) in STATIC_CODES else "<nvrtc>"
    return ("horner_encode_packed_kernel" if packed else "horner_encode_row_kernel") + tag


ENCODE_CODES = [(2, 1), (3, 1), (3, 2), (4, 2), (4, 3), (5, 4),            # static cluster codes
                (1, 1), (6, 4), (6, 5), (7, 6), (8, 8),                    # NVRTC-specialised d <= 8
                (9, 3), (10, 2), (11, 1), (12, 8), (17, 3), (24, 8),       # bit-plane d > 8
                (25, 8), (32, 1), (32, 8)]                                 # d + p > 32: up to d = 32, p = 8


def encode_lengths(d):
    """1, 15-17; unaligned shards in 16-byte payload rows; aligned shards; 31-33, 256 and 257 columns; >= 64 KB"""
    step = 16 // np.gcd(d, 16)                       # d*L % 16 == 0 <=> step | L
    out = {1, 15, 16, 17, 64, 16 * 31, 16 * 32, 16 * 33, 16 * 256, 16 * 257, 16 * 257 - 3, 65536 + 48, 65536 + 7}
    if step < 16:
        out |= {3 * step, 16 * 40 + step}
    return sorted(out)


ENCODE_CASES = [(d, p, L) for d, p in ENCODE_CODES for L in encode_lengths(d)]


def test_encode_matrix_reaches_every_flavour():
    """the matrix below reaches every kernel the single-codeword encode can launch"""
    seen = {predict_encode_kernel(d, p, L) for d, p, L in ENCODE_CASES}
    want = {"rs32_encode_row_kernel", "rs32_encode_row_kernel<segmented>", "rs32_encode_uniform_kernel",
            "horner_encode_row_kernel<static code>", "horner_encode_packed_kernel<static code>",
            "horner_encode_row_kernel<nvrtc>", "horner_encode_packed_kernel<nvrtc>",
            "horner_encode_uniform_kernel", "generic_encode_uniform_kernel"}
    assert seen == want


def _check_encode(rs, oracle, d, p, L, seed):
    rng = np.random.default_rng(seed)
    dbuf, data = _data_slices(d, L, rng)
    pbuf, par, offs = _parity_slices(p, L, fill=GARBAGE)
    dkeep = dbuf.copy()
    rc = rs.lib.ss_rs_encode(rs.h, _ptrs(data + par), d + p, L)
    assert rc == 0, (d, p, L, rc, _err())
    want = _oracle_parity(oracle, d, p, data)
    exp = np.full_like(pbuf, CANARY)
    for o, w in zip(offs, want):
        exp[o:o + L] = w
    assert np.array_equal(dbuf, dkeep), "data shards or their gaps changed"
    for j in range(p):
        assert np.array_equal(par[j], want[j]), (d, p, L, j)
    assert np.array_equal(pbuf, exp), "a canary byte between the parity shards changed"
    return data, par


@pytest.mark.parametrize("d,p", ENCODE_CODES)
def test_encode_single_codeword(coder, oracle, d, p):
    rs = coder(d, p)
    for L in encode_lengths(d):
        _check_encode(rs, oracle, d, p, L, seed=d * 1000 + p * 10 + L)
        assert rs.last_kernel() == predict_encode_kernel(d, p, L), (d, p, L, rs.last_kernel())


@pytest.mark.parametrize("d,p", [(10, 9), (33, 1), (200, 56)])
def test_encode_and_verify_refuse_codes_past_the_kernels(ctx, oracle, d, p):
    """valid crate codes the encoder does not cover: the coder exists, encode / verify refuse and write nothing"""
    rs = ReedSolomon(ctx, d, p)
    assert oracle.rs_new_rc(d, p) == 0
    L = 33
    rng = np.random.default_rng(d)
    dbuf, data = _data_slices(d, L, rng)
    pbuf, par, _ = _parity_slices(p, L, fill=GARBAGE)
    dkeep, pkeep = dbuf.copy(), pbuf.copy()
    rc = rs.lib.ss_rs_encode(rs.h, _ptrs(data + par), d + p, L)
    assert rc == _lib.SS_ERR_UNSUPPORTED and f"coder is {d},{p}" in _err()
    assert np.array_equal(dbuf, dkeep) and np.array_equal(pbuf, pkeep)
    ok = C.c_int(-7)
    rc = rs.lib.ss_rs_verify(rs.h, _ptrs(data + par), d + p, L, C.byref(ok))
    assert rc == _lib.SS_ERR_UNSUPPORTED and f"coder is {d},{p}" in _err() and ok.value == -7
    assert np.array_equal(dbuf, dkeep) and np.array_equal(pbuf, pkeep)
    rs.close()


# ---------------------------------------------------------------------------------------------------------------------
# B. both sides of the staging limit, and grow-only staging
# ---------------------------------------------------------------------------------------------------------------------
def _encode_bytes(d, p, L):
    return d * L + p * round_up(L, 16)


def _reconstruct_bytes(d, p, L):
    return 256 + (d + p) * round_up(L, 16)


def _sides(size, d, row):
    """(largest L that stages, smallest L that does not), both with d*L % 16 == 0 iff row"""
    lo, hi = 1, STAGED_CALL_LIMIT                    # size() grows with L: the last L that stages
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if size(mid) <= STAGED_CALL_LIMIT else (lo, mid - 1)
    hi = lo + 1
    while ((d * lo) % 16 == 0) != row:
        lo -= 1
    while ((d * hi) % 16 == 0) != row:
        hi += 1
    assert size(lo) <= STAGED_CALL_LIMIT < size(hi)
    return lo, hi


def _check_reconstruct_one(rs, oracle, d, p, cw, missing, data_only):
    """one reconstruct call with `missing` shards erased; missing parity of reconstruct_data aliases one buffer"""
    t, L = cw.shape
    alias = np.full(L + 16, CANARY, dtype=np.uint8)
    bufs = []
    for j in range(t):
        b = np.full(L + 3, CANARY, dtype=np.uint8)[1:1 + L]
        b[:] = GARBAGE if j in missing else cw[j]
        bufs.append(b)
    ptr_bufs = [alias[8:8 + L] if (data_only and j >= d and j in missing) else bufs[j] for j in range(t)]
    present = np.array([0 if j in missing else 1 for j in range(t)], dtype=np.uint8)
    fn = rs.lib.ss_rs_reconstruct_data if data_only else rs.lib.ss_rs_reconstruct
    rc = fn(rs.h, _ptrs(ptr_bufs), present.ctypes.data, t, L)
    want_rc, want_pres = _oracle_reconstruct(oracle, d, p, [np.ascontiguousarray(x) for x in cw], present, data_only)
    assert rc == want_rc, (rc, _err())
    assert np.array_equal(present, want_pres)
    upto = d if data_only else t
    for j in range(t):
        want = cw[j] if (j not in missing or j < upto) else np.full(L, GARBAGE, np.uint8)
        assert np.array_equal(bufs[j], want), j
        assert bufs[j].base[0] == CANARY and bufs[j].base[-2:].tolist() == [CANARY, CANARY]
    assert (alias == CANARY).all(), "reconstruct_data touched a missing parity entry"


def _check_encode_reconstruct_verify(rs, oracle, d, p, L, seed):
    data, par = _check_encode(rs, oracle, d, p, L, seed)
    cw = np.stack([np.asarray(s) for s in data + par])
    _check_reconstruct_one(rs, oracle, d, p, cw, {0, d + p - 1}, False)
    _check_reconstruct_one(rs, oracle, d, p, cw, {d - 1, d}, True)
    ok = C.c_int(-1)
    assert rs.lib.ss_rs_verify(rs.h, _ptrs(list(cw)), d + p, L, C.byref(ok)) == 0 and ok.value == 1


@pytest.mark.parametrize("d,p", [(3, 2), (4, 3)])
@pytest.mark.parametrize("row", [True, False])
def test_staging_limit_both_sides(coder, oracle, d, p, row):
    rs = coder(d, p)
    for L in _sides(lambda x: _encode_bytes(d, p, x), d, row):
        _check_encode(rs, oracle, d, p, L, seed=L)
        assert rs.last_kernel() == predict_encode_kernel(d, p, L)
    for L in _sides(lambda x: _reconstruct_bytes(d, p, x), d, row):
        data, par = _check_encode(rs, oracle, d, p, L, seed=L + 1)
        cw = np.stack([np.asarray(s) for s in data + par])
        _check_reconstruct_one(rs, oracle, d, p, cw, {0, d + p - 1}, False)
        _check_reconstruct_one(rs, oracle, d, p, cw, {1, d}, True)


def test_staging_grows_on_one_context(oracle):
    """small, ~24 MiB, small again on a fresh context: the pinned staging and device scratch grow and stay correct"""
    c = Context(0, own_stream=True)
    try:
        rs = ReedSolomon(c, 3, 2)
        big = (24 << 20) // 5 + 5
        for L in (100, big, 100, 4097):
            _check_encode_reconstruct_verify(rs, oracle, 3, 2, L, seed=L)
        rs.close()
    finally:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------
# C. ss_rs_reconstruct / ss_rs_reconstruct_data: every present pattern
# ---------------------------------------------------------------------------------------------------------------------
RECONSTRUCT_KERNEL = {(2, 1): "rs_reconstruct_small_kernel(smem programs)", (3, 2): "rs_reconstruct_small_kernel(smem programs)",
                      (4, 4): "rs_reconstruct_small_kernel", (4, 8): "rs_reconstruct_small_kernel",
                      (5, 4): "horner_reconstruct_kernel", (6, 4): "horner_reconstruct_kernel", (8, 4): "horner_reconstruct_kernel",
                      (9, 3): "generic_reconstruct_kernel", (11, 1): "generic_reconstruct_kernel"}


@functools.lru_cache(maxsize=None)
def _oracle_pattern_table(d, p, data_only):
    """rc and final present[] of the oracle for every present mask (they do not depend on the bytes)"""
    from oracle import pyoracle as oracle
    t = d + p
    cw = _codeword(oracle, d, p, 1, seed=5)
    rcs, press = [], []
    for pat in range(1 << t):
        present = np.array([(pat >> j) & 1 for j in range(t)], dtype=np.uint8)
        bufs = [cw[j].copy() if present[j] else np.zeros(1, np.uint8) for j in range(t)]
        rc, pres = _oracle_reconstruct(oracle, d, p, bufs, present, data_only)
        rcs.append(rc)
        press.append(pres)
    return np.array(rcs), np.stack(press)


@pytest.mark.parametrize("d,p", list(RECONSTRUCT_KERNEL))
@pytest.mark.parametrize("data_only", [False, True])
def test_reconstruct_every_pattern(coder, oracle, d, p, data_only):
    rs = coder(d, p)
    t = d + p
    upto = d if data_only else t
    fn = rs.lib.ss_rs_reconstruct_data if data_only else rs.lib.ss_rs_reconstruct
    pats = np.arange(1 << t)
    bits = ((pats[:, None] >> np.arange(t)) & 1).astype(bool)            # [pattern, shard]
    want_rc, want_pres = _oracle_pattern_table(d, p, data_only)
    assert set(want_rc.tolist()) <= {0, -10}
    sample = set(np.random.default_rng(t).choice(len(pats), min(24, len(pats)), replace=False).tolist())
    for L in (1, 17, 4097, 16 * 65 + 3):
        cw = _codeword(oracle, d, p, L, seed=L * 7 + t)
        Lp = L + 8                                                    # slot + canary tail
        full = np.full((t, Lp), CANARY, dtype=np.uint8)
        full[:, :L] = cw
        garb = full.copy()
        garb[:, :L] = GARBAGE
        work = np.empty_like(full)
        alias = np.full(L + 8, CANARY, dtype=np.uint8)
        rows = [work[j].ctypes.data for j in range(t)]
        arr = (C.c_void_p * t)(*rows)
        present = np.empty(t, dtype=np.uint8)
        reached = False
        for pat in pats:
            pm = bits[pat]
            np.copyto(work, np.where(pm[:, None], full, garb))
            present[:] = pm
            if data_only:                              # the INTEGRATION.md shim: missing parity -> one shared scratch
                for j in range(d, t):
                    arr[j] = rows[j] if pm[j] else alias.ctypes.data
            rc = fn(rs.h, arr, present.ctypes.data, t, L)
            assert rc == want_rc[pat], (L, pat, rc, _err())
            assert np.array_equal(present, want_pres[pat]), (L, pat)
            if rc == 0:
                regen = ~pm & (np.arange(t) < upto)
                exp = np.where((pm | regen)[:, None], full, garb)
                reached = reached or regen.any()
                if regen.any():
                    assert rs.last_kernel() == RECONSTRUCT_KERNEL[(d, p)]
            else:
                exp = np.where(pm[:, None], full, garb)                 # refused: nothing written
            assert np.array_equal(work, exp), (L, pat)
            if L <= 17 or pat in sample:                              # the oracle's own bytes for this pattern
                obufs = [np.ascontiguousarray(np.where(pm[j], full[j, :L], GARBAGE).astype(np.uint8)) for j in range(t)]
                orc, _ = _oracle_reconstruct(oracle, d, p, obufs, pm.astype(np.uint8), data_only)
                assert orc == rc
                for j in range(upto):
                    assert np.array_equal(work[j, :L], obufs[j]), (L, pat, j)
        assert (alias == CANARY).all(), "reconstruct_data read into or wrote a missing parity entry"
        assert reached


@pytest.mark.parametrize("d,p", [(7, 6), (9, 4), (12, 8)])
def test_reconstruct_past_twelve_shards(coder, oracle, d, p):
    """codes with d + p > 12 (RSPaxos at 13 replicas, Crossword-sized codes) have no reconstruct kernel: the calls do
    what needs no kernel and refuse the rest without writing"""
    rs = coder(d, p)
    t = d + p
    L = 37
    cw = _codeword(oracle, d, p, L, seed=t)
    rng = np.random.default_rng(t)
    cases = [set(), set(range(p + 1)), set(range(d, t)), {d}, {t - 1, d + 1}, {0}, {1, d}, {d - 1, t - 1}]
    cases += [set(rng.choice(t, int(rng.integers(1, p + 1)), replace=False).tolist()) for _ in range(6)]
    for missing in cases:
        for data_only in (False, True):
            bufs = [np.full(L, GARBAGE, np.uint8) if j in missing else cw[j].copy() for j in range(t)]
            present = np.array([0 if j in missing else 1 for j in range(t)], dtype=np.uint8)
            pres0 = present.copy()
            fn = rs.lib.ss_rs_reconstruct_data if data_only else rs.lib.ss_rs_reconstruct
            rc = fn(rs.h, _ptrs(bufs), present.ctypes.data, t, L)
            orc, opres = _oracle_reconstruct(oracle, d, p, [b.copy() for b in bufs], pres0, data_only)
            upto = d if data_only else t
            if len(missing) > p:
                want = _lib.SS_ERR_TOO_FEW_SHARDS_PRESENT
            elif not any(j < upto for j in missing):
                want = 0                                               # nothing to regenerate: the oracle's Ok
                assert orc == 0 and np.array_equal(present, opres)
            else:
                want = _lib.SS_ERR_UNSUPPORTED
                assert _err()
            if want != _lib.SS_ERR_UNSUPPORTED:
                assert orc == want
            assert rc == want, (missing, data_only, rc, _err())
            assert np.array_equal(present, pres0)
            for j in range(t):
                assert np.array_equal(bufs[j], np.full(L, GARBAGE, np.uint8) if j in missing else cw[j])


# ---------------------------------------------------------------------------------------------------------------------
# D. ss_rs_verify
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,p", [(2, 1), (3, 2), (4, 3), (6, 4), (8, 8), (9, 3), (12, 8), (32, 8)])
def test_verify(coder, oracle, d, p):
    rs = coder(d, p)
    t = d + p
    lens = (1, 17, 4097) + ((16 * 300,) if (d, p) == (3, 2) else ())
    for L in lens:
        cw = _codeword(oracle, d, p, L, seed=L + t)
        bufs = [np.ascontiguousarray(x.copy()) for x in cw]

        def verify():
            keep = [b.copy() for b in bufs]
            ok = C.c_int(-1)
            rc = rs.lib.ss_rs_verify(rs.h, _ptrs(bufs), t, L, C.byref(ok))
            orc, ook = oracle.rs_verify(d, p, bufs)
            assert rc == orc == 0 and ok.value == int(ook), (L, rc, ok.value, ook)
            assert all(np.array_equal(a, b) for a, b in zip(bufs, keep)), "verify changed a shard"
            return bool(ok.value)
        assert verify()
        flips = [(d + j, k) for j in range(p) for k in sorted({0, L // 2, L - 1})] + [(0, L // 2), (d - 1, L - 1)]
        for j, k in flips:
            for bit in (0, 7):
                bufs[j][k] ^= 1 << bit
                assert not verify(), (L, j, k, bit)
                bufs[j][k] ^= 1 << bit
        # reconstruct -> verify round trip
        if t <= 12:
            missing = {0, t - 1} if p >= 2 else {0}
            for j in missing:
                bufs[j][:] = GARBAGE
            present = np.array([0 if j in missing else 1 for j in range(t)], dtype=np.uint8)
            assert rs.lib.ss_rs_reconstruct(rs.h, _ptrs(bufs), present.ctypes.data, t, L) == 0
            assert verify()
        ok = C.c_int(-1)
        assert rs.lib.ss_rs_verify(rs.h, _ptrs(bufs[:-1]), t - 1, L, C.byref(ok)) == _lib.SS_ERR_TOO_FEW_SHARDS
        assert rs.lib.ss_rs_verify(rs.h, _ptrs(bufs + bufs[:1]), t + 1, L, C.byref(ok)) == _lib.SS_ERR_TOO_MANY_SHARDS
        assert ok.value == -1


# ---------------------------------------------------------------------------------------------------------------------
# E. host-buffer batch calls
# ---------------------------------------------------------------------------------------------------------------------
class _HostMem:
    """numpy views of pageable or ss_host_alloc-pinned host memory"""

    def __init__(self, ctx, pinned):
        self.ctx, self.pinned, self.ptrs = ctx, pinned, []

    def alloc(self, nbytes):
        if not self.pinned:
            return np.empty(nbytes, dtype=np.uint8)
        p = C.c_void_p()
        _lib.check(self.ctx.lib.ss_host_alloc(self.ctx.h, nbytes, C.byref(p)))
        self.ptrs.append(p.value)
        return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p.value))

    def free(self):
        for p in self.ptrs:
            self.ctx.lib.ss_host_free(self.ctx.h, p)
        self.ptrs = []


HOST_CODES = [(3, 2), (4, 3), (6, 4), (12, 8)]
HOST_CASES = [(d, p, ds_kind, ss_kind) for d, p in HOST_CODES for ds_kind in ("ru16", "len", "len+1")
              for ss_kind in ("ru16", "L", "L+5")]


def _host_kernel_ok(d, p, name):
    if (d, p) == (3, 2):
        return name.startswith("rs32_encode_row_kernel")
    if d > 8:
        return name == "generic_encode_uniform_kernel"
    return name.startswith("horner_encode_") and ("<static code>" if (d, p) in STATIC_CODES else "<nvrtc>") in name


@pytest.mark.parametrize("d,p,ds_kind,ss_kind", HOST_CASES)
def test_host_batch_calls(ctx, coder, oracle, monkeypatch, d, p, ds_kind, ss_kind):
    monkeypatch.setenv("SS_E2E_CHUNK_MB", "1")
    rs = coder(d, p)
    i = HOST_CASES.index((d, p, ds_kind, ss_kind))
    n_kind = ("one", "odd_last", "clamp")[i % 3]
    R = (1, 5, 16)[(i // 3) % 3]
    with_bar = i % 2 == 0
    pinned = (i // 2) % 2 == 1
    data_len = (1 << 20) + 1 if n_kind == "clamp" else 999             # odd: data_stride == len is a 2-D upload
    stride = {"ru16": round_up(data_len, 16), "len": data_len, "len+1": data_len + 1}[ds_kind]
    C_chunk = max(2, (1 << 20) // stride) & ~1
    n = {"one": 1, "odd_last": 2 * C_chunk + 3, "clamp": 5}[n_kind]
    L = shard_len(data_len, d)
    ds = round_up(L, 16)
    ss = {"ru16": ds, "L": L, "L+5": L + 5}[ss_kind]
    ps = n * ss + 48                                                    # plane_stride > n * shard_stride
    slot = ds if ss == ds else L
    rng = np.random.default_rng(i)
    mem = _HostMem(ctx, pinned)
    try:
        payload = rng.integers(0, 256, (n, data_len), dtype=np.uint8)
        rows = np.full((n, stride), CANARY, dtype=np.uint8)
        rows[:, :data_len] = payload
        data = mem.alloc((n - 1) * stride + data_len)                  # ends exactly at the last payload
        data[:] = rows.reshape(-1)[:data.size]
        data_keep = data.copy()
        want = oracle.rs_encode_uniform(d, p, payload, data_len)       # [p, n, ds], zero past L
        exp = np.full(p * ps + 32, CANARY, dtype=np.uint8)
        for j in range(p):
            exp[j * ps:j * ps + n * ss].reshape(n, ss)[:, :slot] = want[j, :, :slot]
        planes = mem.alloc(R * n * 8).view(np.uint64).reshape(R, n)
        planes[:] = rng.integers(0, 1 << 63, (R, n), dtype=np.uint64) | rng.integers(0, 1 << 63, (R, n), dtype=np.uint64)
        planes[0] = ~np.uint64(0)
        thr = R // 2 + 1
        c_want, b_want = oracle.tally_planes(planes, thr)
        for fused in (False, True):
            par = mem.alloc(exp.size)
            par[:] = CANARY
            if fused:
                cm = mem.alloc((n + 4) * 8).view(np.uint64)
                cm[:] = 0x1111111111111111
                bar = mem.alloc((n + 4) * 4).view(np.uint32)
                bar[:] = 0x22222222
                rc = rs.lib.ss_accept_step_fused(rs.h, data.ctypes.data, stride, data_len, n, par.ctypes.data, ps, ss,
                                                 planes.ctypes.data, R, thr, cm[2:].ctypes.data,
                                                 bar[2:].ctypes.data if with_bar else None)
            else:
                rc = rs.lib.ss_rs_encode_uniform(rs.h, data.ctypes.data, stride, data_len, n, par.ctypes.data, ps, ss)
            assert rc == 0, _err()
            assert _host_kernel_ok(d, p, rs.last_kernel()), rs.last_kernel()
            if not np.array_equal(par, exp):
                bad = np.flatnonzero(par != exp)
                pytest.fail(f"fused={fused}: {bad.size} host parity bytes differ, first at {bad[0]} "
                            f"(plane {bad[0] // ps}, offset {bad[0] % ps})")
            assert np.array_equal(data, data_keep)
            if fused:
                assert np.array_equal(cm[2:n + 2], c_want)
                assert (cm[:2] == 0x1111111111111111).all() and (cm[n + 2:] == 0x1111111111111111).all()
                if with_bar:
                    assert np.array_equal(bar[2:n + 2], b_want)
                    assert (bar[:2] == 0x22222222).all() and (bar[n + 2:] == 0x22222222).all()
                else:
                    assert (bar == 0x22222222).all()
    finally:
        mem.free()


# ---------------------------------------------------------------------------------------------------------------------
# F. interleaving on one context, threads
# ---------------------------------------------------------------------------------------------------------------------
def test_queued_batch_reconstruct_then_single_codeword_calls(oracle):
    """a (4,3) uniform batch reconstruct keeps its offsets in the context scratch; single-codeword calls right after
    it, without a synchronise in between, first grow that scratch and then reuse it"""
    dev = "cuda:0"
    c = Context(0)                                   # on torch's current stream, fresh scratch
    try:
        d, p, data_len, n = 4, 3, 1000, 20000
        rs = ReedSolomon(c, d, p)
        rng = np.random.default_rng(3)
        payload = rng.integers(0, 256, (n, data_len), dtype=np.uint8)
        L = shard_len(data_len, d)
        ds = round_up(L, 16)
        full = np.zeros((d + p, n, ds), dtype=np.uint8)
        padded = np.zeros((n, d * L), dtype=np.uint8)
        padded[:, :data_len] = payload
        for i in range(d):
            full[i, :, :L] = padded[:, i * L:(i + 1) * L]
        full[d:] = oracle.rs_encode_uniform(d, p, payload, data_len)
        present = rng.integers(0, 1 << (d + p), n).astype(np.uint32)
        damaged = full.copy()
        for j in range(d + p):
            damaged[j][((present >> j) & 1) == 0] = GARBAGE
        sh = torch.from_numpy(damaged).to(dev)
        pm = torch.from_numpy(present.view(np.int32)).to(dev)
        torch.cuda.synchronize()
        st = rs.reconstruct_uniform(sh, data_len, pm, False)          # queued, not synchronised
        _check_encode(rs, oracle, d, p, 400_000, seed=1)            # grows the scratch
        _check_encode(rs, oracle, d, p, 4097, seed=2)               # reuses it
        torch.cuda.synchronize()
        npres = np.array([bin(int(x)).count("1") for x in present])
        assert np.array_equal(st.cpu().numpy(), np.where(npres >= d, 0, -10))
        got = sh.cpu().numpy()
        ok = npres >= d
        assert np.array_equal(got[:, ok, :L], full[:, ok, :L])
        assert np.array_equal(got[:, ~ok], damaged[:, ~ok])
        rs.close()
    finally:
        c.close()


def test_failed_cuda_call_does_not_fail_the_next_call(ctx, coder, oracle):
    """a CUDA runtime error is reported by the call that met it only (here cudaFree of a pointer that is not a device
    allocation, an argument error): the next call on the same thread launches its kernel and succeeds"""
    not_device_memory = np.zeros(64, dtype=np.uint8)
    assert ctx.lib.ss_dev_free(ctx.h, not_device_memory.ctypes.data) == _lib.SS_ERR_CUDA and "cudaFree" in _err()
    _check_encode(coder(4, 3), oracle, 4, 3, 4096, seed=9)
    assert coder(4, 3).last_kernel() == predict_encode_kernel(4, 3, 4096)


THREAD_CODES = [(3, 2), (4, 3), (2, 1), (5, 4), (9, 3)]


def _thread_jobs(oracle, seed, count):
    """random (code, L, op) single-codeword calls with their oracle answers, prepared before the threads start"""
    rng = np.random.default_rng(seed)
    jobs = []
    for _ in range(count):
        d, p = THREAD_CODES[int(rng.integers(len(THREAD_CODES)))]
        t = d + p
        L = int(rng.choice([1, 16, 17, 100, 512, 4097, int(rng.integers(1, 9000))]))
        op = ("encode", "reconstruct", "reconstruct_data", "verify")[int(rng.integers(4))]
        cw = _codeword(oracle, d, p, L, seed=int(rng.integers(1 << 30)))
        missing = set(rng.choice(t, int(rng.integers(1, p + 1)), replace=False).tolist())
        flip = None
        if op == "verify" and rng.integers(2):
            flip = (int(rng.integers(t)), int(rng.integers(L)))
        jobs.append((d, p, L, op, cw, missing, flip))
    return jobs


def _run_job(rs, job):
    d, p, L, op, cw, missing, flip = job
    t = d + p
    if op == "encode":
        bufs = [cw[i].copy() for i in range(d)] + [np.full(L, GARBAGE, np.uint8) for _ in range(p)]
        _lib.check(rs.lib.ss_rs_encode(rs.h, _ptrs(bufs), t, L))
        return all(np.array_equal(bufs[j], cw[j]) for j in range(t))
    if op == "verify":
        bufs = [cw[j].copy() for j in range(t)]
        if flip:
            bufs[flip[0]][flip[1]] ^= 0x10
        ok = C.c_int(-1)
        _lib.check(rs.lib.ss_rs_verify(rs.h, _ptrs(bufs), t, L, C.byref(ok)))
        return ok.value == (0 if flip else 1)
    data_only = op == "reconstruct_data"
    bufs = [np.full(L, GARBAGE, np.uint8) if j in missing else cw[j].copy() for j in range(t)]
    present = np.array([0 if j in missing else 1 for j in range(t)], dtype=np.uint8)
    fn = rs.lib.ss_rs_reconstruct_data if data_only else rs.lib.ss_rs_reconstruct
    _lib.check(fn(rs.h, _ptrs(bufs), present.ctypes.data, t, L))
    upto = d if data_only else t
    return all(np.array_equal(bufs[j], cw[j] if (j not in missing or j < upto) else np.full(L, GARBAGE, np.uint8))
               for j in range(t))


def test_threads_each_with_own_context(oracle):
    """four threads, each with its own context (own stream) and coders, run single-codeword calls concurrently"""
    n_threads = 4
    jobs = [_thread_jobs(oracle, 100 + k, 250) for k in range(n_threads)]
    failures, errors = [], []
    start = threading.Barrier(n_threads)

    def worker(k):
        try:
            c = Context(0, own_stream=True)
            coders = {dp: ReedSolomon(c, *dp) for dp in THREAD_CODES}
            start.wait()
            for idx, job in enumerate(jobs[k]):
                if not _run_job(coders[job[:2]], job):
                    failures.append((k, idx, job[:4]))
            for rs in coders.values():
                rs.close()
            c.close()
        except Exception as e:                      # noqa: BLE001 - reported below
            errors.append((k, repr(e)))
    ts = [threading.Thread(target=worker, args=(k,)) for k in range(n_threads)]
    for th in ts:
        th.start()
    for th in ts:
        th.join()
    assert not errors, errors
    assert not failures, failures[:5]


def test_threads_read_their_own_last_error(ctx, coder):
    """two threads fail with different errors at the same time; each reads its own ss_last_error text"""
    rs = coder(3, 2)
    L = 8
    bufs = [np.zeros(L, np.uint8) for _ in range(5)]
    arr = _ptrs(bufs)
    start = threading.Barrier(2)
    bad = []

    def worker(kind):
        lib = _lib.load()
        start.wait()
        for _ in range(2000):
            if kind == "few":
                rc = lib.ss_rs_encode(rs.h, arr, 4, L)
                want_rc, want_text = _lib.SS_ERR_TOO_FEW_SHARDS, "too few shards"
            else:
                rc = lib.ss_rs_encode(rs.h, arr, 5, 0)
                want_rc, want_text = _lib.SS_ERR_EMPTY_SHARD, "empty shard"
            text = lib.ss_last_error().decode()
            if rc != want_rc or want_text not in text:
                bad.append((kind, rc, text))
    ts = [threading.Thread(target=worker, args=(k,)) for k in ("few", "empty")]
    for th in ts:
        th.start()
    for th in ts:
        th.join()
    assert not bad, bad[:5]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_device1_coder_from_a_device0_thread(oracle):
    c1 = Context(1, own_stream=True)
    try:
        rs = ReedSolomon(c1, 4, 3)
        jobs = _thread_jobs(oracle, 7, 40)
        jobs = [j for j in jobs if j[:2] == (4, 3)] or [(4, 3, 17, "encode", _codeword(oracle, 4, 3, 17, 1), {0}, None)]
        res = []

        def worker():
            torch.cuda.set_device(0)
            res.extend(_run_job(rs, j) for j in jobs)
        th = threading.Thread(target=worker)
        th.start()
        th.join()
        assert res and all(res)
        rs.close()
    finally:
        c1.close()
