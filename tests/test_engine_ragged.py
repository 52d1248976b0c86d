"""Ragged proposals for the RSPaxos / Crossword engine (ss_engine_propose_ragged, summerset_b200/csrc/engine.cu) and
their Accept frames (ss_frame_accept_pack_ragged_dev, summerset_b200/csrc/wire_kernels.cu), against the CPU oracle.

A group's request batch has whatever length ExternalApi::get_req_batch drained (server/external.rs:323-345), and
handle_req_batch codes it as it is (rspaxos/request.rs:72, crossword/request.rs:82): data_len and shard_len differ per
instance, a group with nothing to send proposes nothing.  The engine places each proposing group's shards in a
caller-owned store at 32-byte slot pitches (exclusive scan on the device), runs the ragged encoder once and moves the
instance to Accepting at the group's first Null slot; the packer frames those codewords back to back.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from summerset_b200 import _lib
from summerset_b200 import workloads as wl
from summerset_b200._lib import SummersetError
from tests.test_engine_window import REPLY, _frame, _Model, _reply_frames, _ring_to_window, _tally_fn

DEV = "cuda:0"
U64MAX = np.uint64(0xFFFF_FFFF_FFFF_FFFF)
FRAME_OVERFLOW, WINDOW_FULL, STORE_FULL = 4, 8, 16


def _t(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a).to(DEV)


def _u64(t):
    return t.cpu().numpy().view(np.uint64)


def _pitch(lens, d):
    L = (lens.astype(np.uint64) + np.uint64(d - 1)) // np.uint64(d)
    return np.where(lens > 0, (L + np.uint64(31)) // np.uint64(32) * np.uint64(32), np.uint64(0)).astype(np.uint64)


def _excl_cumsum(x):
    c = np.cumsum(x.astype(np.uint64), dtype=np.uint64)
    return (c - x.astype(np.uint64)).astype(np.uint64), np.uint64(c[-1])


def _ranges(starts, counts):
    starts = np.asarray(starts, dtype=np.int64)
    counts = np.asarray(counts, dtype=np.int64)
    first = np.cumsum(counts) - counts
    return np.arange(int(counts.sum()), dtype=np.int64) + np.repeat(starts - first, counts)


def _arena(rng, lens):
    """payloads after random 0..31-byte gaps: every start offset mod 16; 16 bytes either side for the kernels' loads"""
    gaps = rng.integers(0, 32, len(lens))
    ends = np.cumsum(lens.astype(np.int64) + gaps)
    data_off = 16 + ends - lens.astype(np.int64)
    arena = rng.integers(0, 256, 16 + int(ends[-1]) + 32, dtype=np.uint8)
    return arena, data_off.astype(np.uint64)


def _expect_store(oracle, d, p, canary, arena, data_off, lens, shard_off, ps):
    """canary + the oracle's shards of every codeword with lens > 0, zero-padded to round_up(L, 16), at shard_off"""
    want = canary.copy()
    live = np.nonzero(lens)[0]
    if len(live) == 0:
        return want
    L = (lens.astype(np.int64) + d - 1) // d
    so = shard_off.astype(np.int64)
    want[:, _ranges(so[live] + L[live], (L[live] + 15) // 16 * 16 - L[live])] = 0
    oracle.rs_encode_batch(d, p, arena, data_off[live], lens[live], want[d:].reshape(-1), ps, shard_off[live])
    for g in live:
        o = int(data_off[g])
        want[:d, so[g]:so[g] + L[g]] = oracle.cw_split(arena[o:o + int(lens[g])].tobytes(), d)
    return want


def _assert_same(got, want):
    if np.array_equal(got, want):
        return
    bad = np.argwhere(got != want)
    j, pos = (int(x) for x in bad[0])
    pytest.fail(f"{len(bad)} bytes differ; first in plane {j} at byte {pos}: got {got[j, pos]:#04x}, want {want[j, pos]:#04x}")


def _engine(ctx, oracle, protocol, G, n, T=0, d=0, f=1, bal=None):
    from summerset_b200.engine import LeaderEngine
    eng = LeaderEngine(ctx, protocol, G, n, f, 1, rs_total_shards=T, rs_data_shards=d)
    eng.set_prepared_ballots(_t(bal if bal is not None else np.arange(1, G + 1, dtype=np.uint64)))
    policies = None
    if protocol == "crossword":
        policies = np.stack([oracle.cw_brr_assignment(n, eng.T, spr) for spr in range(eng.T // n, eng.d + 1, eng.T // n)])
        eng.set_policies([list(map(int, q)) for q in policies], True)
    return eng, policies


def _lengths(rng, d, extra_random=0):
    edges = [0, 0, 1, d - 1, d, 16 * d - 1, 16 * d, 16 * d + 1, 1365, 1366, 1367, 4096, 65536]
    cfg4, _ = wl.cfg4_lengths(64, seed_extra=d)
    lens = np.concatenate([edges, cfg4, rng.integers(1, 3001, extra_random)]).astype(np.uint32)
    rng.shuffle(lens)
    return lens


# ---------------------------------------------------------------------------------------------
# store content: every byte of the caller's store
# ---------------------------------------------------------------------------------------------
# RS(3,2) -> rs32_encode_ragged_kernel; RS(4,3) and RS(6,4) -> horner_encode_ragged_kernel; RS(9,1) ->
# generic_encode_ragged_kernel
CODES = [("rspaxos", 5, 0, 0), ("rspaxos", 7, 0, 0), ("crossword", 5, 5, 3), ("crossword", 5, 10, 6), ("crossword", 5, 10, 9)]


@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,T,d", CODES)
def test_ragged_store_content(ctx, oracle, protocol, n, T, d):
    rng = np.random.default_rng(100 * n + 10 * T + d)
    G0 = len(_lengths(rng, 3, 50))
    eng, policies = _engine(ctx, oracle, protocol, G0, n, T, d)
    d, p = eng.d, eng.T - eng.d
    lens = _lengths(rng, d, 50)
    assert len(lens) == G0
    arena, data_off = _arena(rng, lens)
    pitch = _pitch(lens, d)
    off, need = _excl_cumsum(pitch)
    ps = int(need) + 96
    canary = rng.integers(0, 256, (eng.T, ps), dtype=np.uint8)
    store = _t(canary.copy())
    pol = rng.integers(0, len(policies), G0).astype(np.uint8) if policies is not None else None
    a, do, ln = _t(arena), _t(data_off), _t(lens)
    slot_out, shard_off, need_d = eng.propose_ragged(a, do, ln, store, _t(pol) if pol is not None else None)
    assert ctx.device_status() == 0
    live = lens > 0
    assert (_u64(shard_off)[live] == off[live]).all() and (_u64(shard_off)[~live] == U64MAX).all()
    assert _u64(need_d)[0] == need
    assert (_u64(slot_out)[live] == 0).all() and (_u64(slot_out)[~live] == U64MAX).all()
    _assert_same(store.cpu().numpy(), _expect_store(oracle, d, p, canary, arena, data_off, lens, off, ps))
    assert (_u64(eng.accepting) == live.astype(np.uint64)).all()
    eng.close()


# ---------------------------------------------------------------------------------------------
# offsets and per-group state against a model of first_null_slot
# ---------------------------------------------------------------------------------------------
def _trailing_ones(x):
    y = ~x
    low = y & (~y + np.uint64(1))
    return np.where(y == 0, 64, np.log2(np.maximum(low, np.uint64(1)).astype(np.float64)).astype(np.int64))


def _random_state(rng, eng, G):
    """random window bases, accepting / committed words (some windows full), ack planes, inst_bal, policy_idx"""
    base = rng.integers(0, 1 << 40, G).astype(np.uint64)
    occ = np.where(rng.random(G) < 0.15, U64MAX, rng.integers(0, 1 << 63, G, dtype=np.uint64) & rng.integers(0, 1 << 63, G, dtype=np.uint64))
    split = rng.integers(0, 1 << 63, G, dtype=np.uint64)
    acc, cm = occ & split, occ & ~split
    r = (base & np.uint64(63))
    to_ring = lambda x: (x << r) | (x >> ((np.uint64(64) - r) & np.uint64(63)))
    eng.window_base.copy_(_t(base))
    eng.accepting.copy_(_t(to_ring(acc)))
    eng.committed.copy_(_t(to_ring(cm)))
    eng.planes.copy_(_t(rng.integers(0, 1 << 63, eng.planes.shape, dtype=np.uint64)))
    eng.inst_bal.copy_(_t(rng.integers(0, 1 << 40, G * 64).astype(np.uint64)))
    if eng.policy_idx is not None:
        eng.policy_idx.copy_(_t(rng.integers(0, 3, G * 64).astype(np.uint8)))


def _snapshot(eng):
    torch.cuda.synchronize()
    s = {k: _u64(getattr(eng, k)).copy() for k in ("accepting", "committed", "planes", "inst_bal", "window_base")}
    if eng.policy_idx is not None:
        s["policy_idx"] = eng.policy_idx.cpu().numpy().copy()
    return s


def _apply_model(before, bal, proposing, pol):
    """the state after group g (proposing[g]) entered Accepting at its first Null slot; returns (state, slot_out)"""
    want = {k: v.copy() for k, v in before.items()}
    base = before["window_base"]
    r = base & np.uint64(63)
    occ_w = _ring_to_window(before["accepting"] | before["committed"], base)
    rel = _trailing_ones(occ_w)
    g = np.nonzero(proposing)[0]
    assert (rel[g] < 64).all()
    s = base[g] + rel[g].astype(np.uint64)
    pos = (s & np.uint64(63)).astype(np.int64)
    bit = np.uint64(1) << pos.astype(np.uint64)
    want["accepting"][g] |= bit
    want["committed"][g] &= ~bit
    want["planes"][:, g] &= ~bit
    want["inst_bal"][g * 64 + pos] = bal[g]
    if "policy_idx" in want:
        want["policy_idx"][g * 64 + pos] = pol[g] if pol is not None else 0
    slot_out = np.full(len(base), U64MAX)
    slot_out[g] = s
    return want, slot_out, rel


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 255, 256, 257, 4099, 1 << 20])
def test_ragged_offsets_and_state(ctx, oracle, G):
    rng = np.random.default_rng(G)
    bal = rng.integers(1, 1 << 40, G).astype(np.uint64)
    eng, policies = _engine(ctx, oracle, "crossword", G, 5, 5, 3, f=1, bal=bal)
    _random_state(rng, eng, G)
    lens = np.where(rng.random(G) < 0.2, 0, rng.integers(1, 300, G)).astype(np.uint32)
    arena, data_off = _arena(rng, lens)
    pol = rng.integers(0, len(policies), G).astype(np.uint8)
    before = _snapshot(eng)
    rel = _trailing_ones(_ring_to_window(before["accepting"] | before["committed"], before["window_base"]))
    proposing = (lens > 0) & (rel < 64)
    pitch = _pitch(np.where(proposing, lens, 0), 3)
    off, need = _excl_cumsum(pitch)
    store = torch.zeros((5, int(need) + 32), dtype=torch.uint8, device=DEV)
    slot_out, shard_off, need_d = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, _t(pol))
    status = ctx.device_status()
    assert status == (WINDOW_FULL if ((lens > 0) & (rel == 64)).any() else 0)
    assert _u64(need_d)[0] == need
    assert (_u64(shard_off) == np.where(proposing, off, U64MAX)).all()
    want, want_slot, _ = _apply_model(before, bal, proposing, pol)
    assert (_u64(slot_out) == want_slot).all()
    got = _snapshot(eng)
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    eng.close()


@pytest.mark.gpu
def test_ragged_skipped_groups_and_store_full(ctx, oracle):
    """data_len == 0 and full windows take no room; a plane_stride too small proposes exactly the prefix of the
    proposing groups that fits, sets SS_DEV_STATUS_STORE_FULL and leaves the rest -- state and store -- unchanged."""
    G = 3000
    rng = np.random.default_rng(31)
    bal = rng.integers(1, 1 << 40, G).astype(np.uint64)
    eng, _ = _engine(ctx, oracle, "rspaxos", G, 5, bal=bal)
    _random_state(rng, eng, G)
    lens = np.where(rng.random(G) < 0.2, 0, rng.integers(1, 5000, G)).astype(np.uint32)
    arena, data_off = _arena(rng, lens)
    before = _snapshot(eng)
    rel = _trailing_ones(_ring_to_window(before["accepting"] | before["committed"], before["window_base"]))
    asked = (lens > 0) & (rel < 64)
    pitch = _pitch(np.where(asked, lens, 0), 3)
    off, need = _excl_cumsum(pitch)
    ps = int(need) // 2 // 32 * 32
    fits = asked & (off + pitch <= np.uint64(ps))
    assert 0 < fits.sum() < asked.sum()
    k = np.nonzero(asked & ~fits)[0][0]                   # the first group that does not fit: all after it fail too
    assert not (fits[k:]).any()
    canary = rng.integers(0, 256, (5, ps), dtype=np.uint8)
    store = _t(canary.copy())
    slot_out, shard_off, need_d = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store)
    assert ctx.device_status() == WINDOW_FULL | STORE_FULL
    assert _u64(need_d)[0] == need
    assert (_u64(shard_off) == np.where(fits, off, U64MAX)).all()
    want, want_slot, _ = _apply_model(before, bal, fits, None)
    assert (_u64(slot_out) == want_slot).all()
    got = _snapshot(eng)
    for key in want:
        assert np.array_equal(got[key], want[key]), key
    _assert_same(store.cpu().numpy(), _expect_store(oracle, 3, 2, canary, arena, data_off, np.where(fits, lens, 0), off, ps))
    # nothing to propose at all: no status, no change
    before = _snapshot(eng)
    slot_out, shard_off, need_d = eng.propose_ragged(_t(arena), _t(data_off), _t(np.zeros(G, np.uint32)), store)
    assert ctx.device_status() == 0 and _u64(need_d)[0] == 0
    assert (_u64(slot_out) == U64MAX).all() and (_u64(shard_off) == U64MAX).all()
    got = _snapshot(eng)
    for key in before:
        assert np.array_equal(got[key], before[key]), key
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("protocol", ["rspaxos", "crossword"])
def test_ragged_equal_lengths_equal_propose_next(ctx, oracle, protocol):
    """All lengths equal: the planes at their slots and the whole engine state equal propose_next's on a twin engine."""
    from summerset_b200.engine import LeaderEngine
    G, n, data_len, k = 700, 5, 2999, 5
    kw = dict(rs_total_shards=5, rs_data_shards=3) if protocol == "crossword" else {}
    twin = LeaderEngine(ctx, protocol, G, n, 1, data_len, **kw)
    eng = LeaderEngine(ctx, protocol, G, n, 1, 1, **kw)
    rng = np.random.default_rng(3)
    for e in (twin, eng):
        e.set_prepared_ballots(_t(np.arange(9, G + 9, dtype=np.uint64)))
        if protocol == "crossword":
            e.set_policies([list(map(int, oracle.cw_brr_assignment(n, 5, spr))) for spr in (1, 2, 3)], True)
    L = -(-data_len // 3)
    ds, pitch = (L + 15) // 16 * 16, (L + 31) // 32 * 32
    lens = _t(np.full(G, data_len, dtype=np.uint32))
    for i in range(k):
        payload = wl.payload_uniform(G, data_len, seed_extra=60 + i)
        pol = _t(rng.integers(0, 3, G).astype(np.uint8)) if protocol == "crossword" else None
        pay = _t(payload)
        want_slot, planes = twin.propose_next(0, pay, pol)
        store = torch.full((5, G * pitch), 0x3C, dtype=torch.uint8, device=DEV)
        offs = _t(np.arange(G, dtype=np.uint64) * np.uint64(payload.shape[1]))
        slot_out, shard_off, need = eng.propose_ragged(pay.reshape(-1), offs, lens, store, pol)
        assert torch.equal(slot_out, want_slot)
        assert (_u64(shard_off) == np.arange(G, dtype=np.uint64) * np.uint64(pitch)).all() and int(need) == G * pitch
        got = store.reshape(5, G, pitch)
        assert torch.equal(got[:, :, :ds], planes)
        assert (got[:, :, ds:] == 0x3C).all()
    names = ["planes", "bal_prepared", "inst_bal", "accepting", "committed", "commit_bar"] + (["policy_idx"] if protocol == "crossword" else [])
    for name in names:
        assert torch.equal(getattr(eng, name), getattr(twin, name)), name
    twin.close()
    eng.close()


# ---------------------------------------------------------------------------------------------
# Accept frames and AcceptData records of a ragged proposal
# ---------------------------------------------------------------------------------------------
def _vlen(v):
    return 1 if v < 251 else 3 if v < 1 << 16 else 5 if v < 1 << 32 else 9


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["rspaxos_accept", "crossword_accept", "wal_accept_data"])
def test_ragged_frames_match_oracle(ctx, oracle, kind):
    rng = np.random.default_rng(len(kind))
    n = 5
    cw = kind == "crossword_accept"
    lens = _lengths(rng, 3, 150)
    G = len(lens)
    bal = rng.integers(1, 1 << 40, G).astype(np.uint64)
    eng, policies = _engine(ctx, oracle, "crossword" if cw else "rspaxos", G, n, 5 if cw else 0, 3 if cw else 0, bal=bal)
    d, p, T = eng.d, eng.T - eng.d, eng.T
    eng.window_base.copy_(_t(rng.integers(0, 1 << 40, G).astype(np.uint64)))
    eng.accepting[: G // 10] = -1                          # full windows: those groups propose nothing
    arena, data_off = _arena(rng, lens)
    pol = rng.integers(0, len(policies), G).astype(np.uint8) if cw else np.zeros(G, np.uint8)
    if not cw:
        policies = np.array([[1 << r for r in range(n)]], dtype=np.uint32)   # replica r holds shard r
    need = int(_excl_cumsum(_pitch(lens, d))[1])
    store = torch.zeros((T, need + 32), dtype=torch.uint8, device=DEV)
    slot_out, shard_off, _ = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, _t(pol) if cw else None)
    assert ctx.device_status() == WINDOW_FULL
    slot, so = _u64(slot_out), _u64(shard_off)
    assert (slot[: G // 10] == U64MAX).all()
    ln_d, pol_d, bal_d = _t(lens), _t(pol), _t(bal)
    wal = kind == "wal_accept_data"
    planes = store.cpu().numpy()
    for peer in range(n):
        out, off, fl, total = ctx.frame_accept_pack_ragged(store, shard_off, ln_d, d, p, policies, pol_d, peer, slot_out, bal_d,
                                                           kind=1 if wal else 0, msg_variant=1 if wal else 2, with_assignment=cw)
        assert ctx.device_status() == 0
        out, off, fl = out.cpu().numpy(), off.cpu().numpy(), fl.cpu().numpy()
        start = 0
        for g in range(G):
            if lens[g] == 0 or slot[g] == U64MAX:
                assert fl[g] == 0
                continue
            L = -(-int(lens[g]) // d)
            mask = int(policies[pol[g]][peer])
            shards = [planes[j, int(so[g]):int(so[g]) + L].tobytes() if (mask >> j) & 1 else None for j in range(T)]
            got = out[int(off[g]):int(off[g]) + int(fl[g])].tobytes()
            if wal:
                want = oracle.wal_accept_data(int(slot[g]), int(bal[g]), d, p, int(lens[g]), shards)
            elif any(s is not None for s in shards):
                want = oracle.frame_accept(2, int(slot[g]), int(bal[g]), d, p, int(lens[g]), shards,
                                           list(map(int, policies[pol[g]])) if cw else None, T)
            else:
                want = None                                # the peer's assignment is empty: no oracle frame to compare
            if want is not None:
                assert got == want, (kind, peer, g)
            dec = oracle.decode_accept(got, 1 if wal else 0, cw)
            assert dec and dec["shards"] == shards and dec["slot"] == int(slot[g]) and dec["data_len"] == int(lens[g])
            assert dec["shard_len"] == L
            # packed regions, the first carried shard's bytes 16-byte aligned
            pad = int(off[g]) - start
            assert 0 <= pad < 16
            if mask:
                h = (0 if wal else 1) + _vlen(1 if wal else 2) + _vlen(int(slot[g])) + _vlen(int(bal[g])) + 2 + \
                    _vlen(int(lens[g])) + _vlen(L) + _vlen(T)
                first = (mask & -mask).bit_length() - 1
                assert (int(off[g]) + 8 + h + first + 1 + _vlen(L)) % 16 == 0
            start += (pad + int(fl[g]) + 15) // 16 * 16
        assert int(total) == start


@pytest.mark.gpu
def test_ragged_frames_skip_and_overflow(ctx, oracle):
    """UINT64_MAX slots and null codewords get no frame; a short out_capacity writes exactly the frames whose regions fit,
    sets SS_DEV_STATUS_FRAME_OVERFLOW, and leaves every other byte of out alone."""
    rng = np.random.default_rng(77)
    G, d, p = 500, 3, 2
    lens = np.where(rng.random(G) < 0.2, 0, rng.integers(1, 9000, G)).astype(np.uint32)
    so = _excl_cumsum(_pitch(lens, d))[0]
    planes = rng.integers(0, 256, (5, int(so[-1]) + 4096), dtype=np.uint8)
    slot = rng.integers(0, 1 << 40, G).astype(np.uint64)
    slot[rng.random(G) < 0.1] = U64MAX
    bal = rng.integers(1, 1 << 40, G).astype(np.uint64)
    policies = [[0b00111, 0b01110, 0b11100, 0b11001, 0b10011]]
    args = (_t(planes), _t(so), _t(lens), d, p, policies, None, 2, _t(slot), _t(bal))
    full, off0, fl0, total = ctx.frame_accept_pack_ragged(*args)
    assert ctx.device_status() == 0
    fl0 = fl0.cpu().numpy()
    skipped = (lens == 0) | (slot == U64MAX)
    assert (fl0[skipped] == 0).all() and (fl0[~skipped] > 0).all()
    cap = int(total) // 2 // 16 * 16 + 5
    out, off, fl, total2 = ctx.frame_accept_pack_ragged(*args, out_capacity=cap)
    assert ctx.device_status() == FRAME_OVERFLOW and int(total2) == int(total)
    out, off, fl, off0, full = out.cpu().numpy(), off.cpu().numpy(), fl.cpu().numpy(), off0.cpu().numpy(), full.cpu().numpy()
    # regions in group order: the region of g ends at the next written frame's region start, or at total
    ends = np.empty(G, dtype=np.int64)
    nxt = int(total)
    for g in range(G - 1, -1, -1):
        ends[g] = nxt
        if not skipped[g]:
            nxt = int(off0[g]) // 16 * 16
    fits = ~skipped & (ends <= cap)
    assert 0 < fits.sum() < (~skipped).sum()
    assert (fl[fits] == fl0[fits]).all() and (fl[~fits] == 0).all() and (off[fits] == off0[fits]).all()
    want = np.full(cap, 0xA5, dtype=np.uint8)
    for g in np.nonzero(fits)[0]:
        want[int(off0[g]):int(off0[g]) + int(fl0[g])] = full[int(off0[g]):int(off0[g]) + int(fl0[g])]
    assert np.array_equal(out, want)


# ---------------------------------------------------------------------------------------------
# round trip: ragged proposals -> AcceptReply frames -> parse -> ingest -> tick -> advance, over several windows
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("protocol", ["rspaxos", "crossword"])
def test_ragged_round_trip_windows(ctx, oracle, protocol):
    G, n, f = 800, 5, 1
    rng = np.random.default_rng(11 if protocol == "rspaxos" else 12)
    bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
    cw = protocol == "crossword"
    eng, policies = _engine(ctx, oracle, protocol, G, n, 5 if cw else 0, 3 if cw else 0, f=f, bal=bal)
    model = _Model(G, bal)
    tally = _tally_fn(oracle, model, protocol, n, f, n // 2 + 1 + f, 5, 3, True, policies)
    weight = np.where(rng.random(G) < 0.2, 0.1, 1.0)
    newly = torch.zeros(G, dtype=torch.int64, device=DEV)
    seen_full = seen_idle = 0
    for rnd in range(40):
        for k in range(int(rng.integers(1, 5))):
            want = model.first_null(oracle)
            lens = np.where(rng.random(G) < 0.2, 0, wl.cfg4_lengths(G, seed_extra=100 * rnd + k)[0] // 16).astype(np.uint32)
            want = np.where(lens > 0, want, -1)
            full = (lens > 0) & (want < 0)
            arena, data_off = _arena(rng, lens)
            pol = rng.integers(0, len(policies), G).astype(np.uint8) if cw else np.zeros(G, np.uint8)
            need = int(_excl_cumsum(_pitch(lens, 3))[1])
            store = torch.empty((5, need + 32), dtype=torch.uint8, device=DEV)
            slot_out, _, _ = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, _t(pol) if cw else None)
            assert ctx.device_status() == (WINDOW_FULL if full.any() else 0)
            got = _u64(slot_out)
            assert (got[want >= 0] == want[want >= 0].astype(np.uint64)).all() and (got[want < 0] == U64MAX).all()
            seen_full += int(full.sum())
            seen_idle += int((lens == 0).sum())
            model.propose(oracle, want, pol)
        for _ in range(2):
            (buf, offs, fg, fp), recs = _reply_frames(oracle, rng, model, n, 16 * G, weight, 0, cw)
            rg, rs_, rp, rb, rk = ctx.accept_reply_parse(_t(buf), _t(offs), _t(fg), _t(fp), eng.window_base, REPLY, cw)
            eng.on_accept_replies(rg, rs_, rp, rb)
            committed, bar = eng.tick(newly)
            torch.cuda.synchronize()
            assert (rk.cpu().numpy() == REPLY).all()
            tally(*recs)
            want_c = model.window(oracle.ST_COMMITTED)
            wb = _u64(eng.window_base)
            assert (_ring_to_window(_u64(committed), wb) == want_c).all(), rnd
            assert (_ring_to_window(_u64(eng.accepting), wb) == model.window(oracle.ST_ACCEPTING)).all(), rnd
            want_bar = np.array([oracle.commit_bar(int(w)) for w in want_c], dtype=np.uint32)
            assert (bar.cpu().numpy().view(np.uint32) == want_bar).all(), rnd
        bar_m = np.array([oracle.commit_bar(int(w)) for w in model.window(oracle.ST_COMMITTED)], dtype=np.int64)
        eng.advance()
        model.mb += bar_m
        torch.cuda.synchronize()
        assert (_u64(eng.window_base) == model.mb.astype(np.uint64)).all(), rnd
    assert model.mb.max() >= 64 and seen_full > 0 and seen_idle > 0 and model.top.max() < 256
    eng.close()


# ---------------------------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ragged_rejects_other_engines_and_bad_strides(ctx):
    from summerset_b200.engine import LeaderEngine, RaftEngine
    dummy = torch.zeros(64, dtype=torch.int64, device=DEV)
    ptr = dummy.data_ptr()
    for e in (LeaderEngine(ctx, "multipaxos", 16, 5), RaftEngine(ctx, 16, 5)):
        assert e.lib.ss_engine_propose_ragged(e.h, ptr, ptr, ptr, None, ptr, 64, ptr, ptr, None) == _lib.SS_ERR_INVALID_ARG
        e.close()
    eng = LeaderEngine(ctx, "rspaxos", 16, 5, 1, 1)
    with pytest.raises(SummersetError) as ei:
        eng.propose_ragged(dummy.view(torch.uint8), dummy[:16], dummy[:8].view(torch.int32),
                           torch.zeros((5, 48), dtype=torch.uint8, device=DEV))
    assert ei.value.code == _lib.SS_ERR_INVALID_ARG
    eng.close()


def test_ragged_calls_reject_null_handles():
    lib = _lib.load()
    assert lib.ss_engine_propose_ragged(None, None, None, None, None, None, 32, None, None, None) == _lib.SS_ERR_INVALID_ARG
    spec = _lib.FrameSpec(0, 2, 3, 2, 0, 5, 0, 5)
    assert lib.ss_frame_accept_pack_ragged_dev(None, C.byref(spec), None, 0, None, None, None, 1, None, 0, None, None, 1, None, 0,
                                               None, None, None) == _lib.SS_ERR_INVALID_ARG
