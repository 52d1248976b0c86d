"""The device acceptor (ss_acceptor_*, summerset_b200/csrc/acceptor.cu) across what its ABI accepts.

tests/test_acceptor.py pins the semantics at population 5 on a few codes; this file runs the same per-message model
(`_stream`) and the same byte-for-byte check (`_run_and_check`) over:
  A  every population 1..32 for RSPaxos and Crossword, T = n and T = 2n, d = 1, d = T, T = 32, T not a multiple of n,
     `me` at 0, n // 2 and n - 1, balanced / unbalanced / empty / full assignment rows, shard lengths at the varint
     edges; frames from the real leader path where the engine takes the code, from the device packer elsewhere
  B  accept / WAL / reply variants of every varint width, and frames of other variants around 2^16
  C  the widest reply cell (42 bytes) and the data_len bound
  D  batch sizes across the scan tiles and past every kernel's grid cap, and an advance past its grid cap
  E  sort keys at and around powers of two
  F  one acceptor over calls that shrink and regrow its scratch
  G  one hot group of 20k frames
  I  a non-blocking context stream while torch's default stream is busy
  J  the AcceptReply parser's frame bounds near the end of the buffer and near 2^64
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pyoracle
from summerset_b200 import _lib
from tests.test_acceptor import (ACC, MALFORMED, U64MAX, Cfg, State, _acceptor, _adversarial, _advance, _buffer, _check_state,
                                 _decode, _install, _leader_frames, _run_and_check, _stream, _t, _vput)

DEV = "cuda:0"
U32MAX = (1 << 32) - 1
VARIANT_EDGES = [0, 250, 251, 65535, 65536, U32MAX]
# (accept_variant, wal_variant, reply_variant): every edge once in every position, widths mixed in each setting
VARIANT_SETTINGS = [tuple(VARIANT_EDGES[(i + k) % 6] for k in range(3)) for i in range(6)]


def _maj(n):
    return n // 2 + 1


# ---------------------------------------------------------------------------------------------
# A: the population x code x me matrix
# ---------------------------------------------------------------------------------------------
def _matrix_codes():
    out = []
    for n in range(1, 33):
        out.append(("rspaxos", n, _maj(n), n))
        out.append(("crossword", n, _maj(n), n))
        if 2 * n <= 32:
            out.append(("crossword", n, n, 2 * n))
    out += [("rspaxos", 5, 1, 5), ("crossword", 8, 1, 8), ("crossword", 3, 1, 6),          # d = 1
            ("rspaxos", 4, 4, 4), ("crossword", 6, 6, 6), ("crossword", 3, 12, 12)]          # d = T: no parity
    out += [("crossword", n, d, 32) for n, d in ((1, 17), (2, 1), (4, 32), (8, 5), (16, 9))]  # T = 32 (n = 32: above)
    out += [("rspaxos", 3, 2, 32), ("crossword", 5, 3, 7), ("crossword", 7, 4, 32), ("crossword", 12, 7, 13)]
    return out


MATRIX = _matrix_codes()


def _mes(n):
    return sorted({0, n // 2, n - 1})


def _engine_takes(protocol, n, d, T):
    """codes LeaderEngine accepts (engine.cu: ss_engine_create) and its batched encoder runs (p <= 8)"""
    if n > 12 or T - d > 8:
        return False
    if protocol == "rspaxos":
        return d == _maj(n) and T == n and T > d
    return T % n == 0 and _maj(n) <= d < T


def _lens(rng, d):
    """request lengths: shard lengths 250, 251, 65535 and 65536 exactly, small ones, and a mix"""
    edges = [L * d for L in (250, 251, 65535, 65536)] + [1, d, d + 1, 249 * d + 1]
    return np.concatenate([edges, rng.integers(1, 3000, 12)]).astype(np.uint32)


def _tables(oracle, rng, cfg, mes):
    """Crossword assignment tables (one row per replica): balanced, unbalanced, an empty row at each `me`, all rows full"""
    n, T, d = cfg.n, cfg.T, cfg.d
    full = (1 << T) - 1
    if not cfg.cw:
        return [[1 << r for r in range(n)]]
    tabs = [[int(x) for x in oracle.cw_brr_assignment(n, T, spr)] for spr in sorted({max(1, T // n), d})]
    tabs.append([int(rng.integers(0, full + 1)) for _ in range(n)])
    for me in mes:
        t = [int(rng.integers(1, full + 1)) for _ in range(n)]
        t[me] = 0
        tabs.append(t)
    tabs.append([full] * n)
    return tabs


def _oracle_accept(oracle, av, slot, ballot, d, p, dlen, shards, asg, T):
    """oracle.frame_accept, also for a frame that carries no shard"""
    L = -(-dlen // d)
    if any(s is not None for s in shards):
        return oracle.frame_accept(av, slot, ballot, d, p, dlen, shards, asg, T)
    arr = (C.c_void_p * len(shards))()
    out = np.zeros(64 + len(shards) + (len(asg) * 24 if asg else 0), dtype=np.uint8)
    a = np.ascontiguousarray(np.array(asg, dtype=np.uint32)) if asg is not None else None
    lib = oracle.lib()
    lib.ssor_frame_accept.restype = C.c_size_t
    n = lib.ssor_frame_accept(av, C.c_uint64(slot), C.c_uint64(ballot), d, p, C.c_uint64(dlen), C.c_uint64(L), arr,
                              None if a is None else C.c_void_p(a.ctypes.data), len(asg) if asg is not None else 0, T,
                              C.c_void_p(out.ctypes.data))
    return out[:n].tobytes()


class _Store:
    """a shard store [T, stride] filled with the oracle's encoding of random requests, as propose_ragged lays it out"""

    def __init__(self, oracle, rng, cfg, lens):
        d, T = cfg.d, cfg.T
        self.lens = lens
        L = (lens.astype(np.int64) + d - 1) // d
        pitch = (L + 31) // 32 * 32
        self.off = np.concatenate([[0], np.cumsum(pitch)[:-1]]).astype(np.int64)
        self.planes = np.zeros((T, int(pitch.sum()) + 32), dtype=np.uint8)
        self.shards = []
        for g, ln in enumerate(lens):
            sh = oracle.cw_split(rng.integers(0, 256, int(ln), dtype=np.uint8).tobytes(), d)
            rows = [np.ascontiguousarray(sh[j]) for j in range(d)] + [np.zeros(int(L[g]), np.uint8) for _ in range(T - d)]
            if T > d:
                assert oracle.rs_encode(d, T - d, rows) == 0
            for j in range(T):
                self.planes[j, self.off[g]:self.off[g] + L[g]] = rows[j]
            self.shards.append([r.tobytes() for r in rows])


def _packed_frames(ctx, oracle, cfg, store, tables, pol, slots, bals, peer):
    """frames for `peer` from ss_frame_accept_pack_ragged_dev, each checked byte for byte against oracle.frame_accept"""
    d, T = cfg.d, cfg.T
    out, off, fl, _ = ctx.frame_accept_pack_ragged(_t(store.planes), _t(store.off), _t(store.lens), d, T - d, tables, _t(pol), peer,
                                                   _t(slots), _t(bals), msg_variant=cfg.av, with_assignment=cfg.cw)
    assert ctx.device_status() == 0
    out, off, fl = out.cpu().numpy(), off.cpu().numpy(), fl.cpu().numpy()
    frames = []
    for g in range(len(store.lens)):
        fr = out[int(off[g]):int(off[g]) + int(fl[g])].tobytes()
        mask = tables[pol[g]][peer]
        shards = [store.shards[g][j] if (mask >> j) & 1 else None for j in range(T)]
        want = _oracle_accept(oracle, cfg.av, int(slots[g]), int(bals[g]), d, T - d, int(store.lens[g]), shards,
                              tables[pol[g]] if cfg.cw else None, T)
        assert fr == want, (g, peer)
        frames.append(fr)
    return frames


def _other_variant_frames(cfg):
    """messages that are not this acceptor's Accept: PeerMsg and PeerMessage variants on both sides of 2^16"""
    out = []
    for v in (3, 65535, 65536, U32MAX):
        if v != cfg.av:
            body = b"\x00" + _vput(v) + _vput(7) + _vput(1)
            out.append(len(body).to_bytes(8, "big") + body)
    for v in (1, 65535, 65536, U32MAX):
        body = _vput(v) + b"\x01"
        out.append(len(body).to_bytes(8, "big") + body)
    return out


def _check_reply_parse(ctx, acc, cfg, want, got, groups, st):
    """every accepted reply cell through ss_accept_reply_parse_dev, against the oracle's parse_accept_reply"""
    idx = [i for i, v in enumerate(want["verdict"]) if v == ACC]
    if not idx:
        return
    cells = got["replies"]
    rg, rs_, rp, rb, rk = ctx.accept_reply_parse(_t(cells.reshape(-1)), _t(np.array([48 * i for i in idx], dtype=np.uint64)),
                                                 _t(np.array([groups[i] for i in idx], dtype=np.uint32)),
                                                 _t(np.zeros(len(idx), np.uint8)), acc.window_base, cfg.rv, cfg.cw)
    rs_, rb, rk = rs_.cpu().numpy(), rb.cpu().numpy().view(np.uint64), rk.cpu().numpy().view(np.uint32)
    for k, i in enumerate(idx):
        f = want["dec"][i]
        n, slot, bal, size, kind = pyoracle.parse_accept_reply(cells[i].tobytes(), cfg.rv, cfg.cw)
        inst = st.inst[groups[i]][f["slot"]]
        assert (n, slot, bal) == (len(want["replies"][i]), f["slot"], inst["bal"]), i
        if cfg.cw:
            assert size == bin(inst["asg"][cfg.me]).count("1") * (inst["dlen"] // cfg.d + 1)
        assert (int(rk[k]), int(rb[k]), int(rs_[k])) == (cfg.rv, bal, slot - st.base[groups[i]]), i


def _matrix_cell(ctx, oracle, cfg, rng, frames, base, n_adv=150, extra=()):
    """frames[g] goes to group g (accepted: inside the window at the group's top ballot); adversarial frames and `extra`
    are mixed in, the batch is shuffled and checked against the model, then every reply is parsed back"""
    G = len(frames) + 4
    acc = _acceptor(ctx, cfg, G)
    st = State(G)
    st.base = [int(x) for x in base] + [int(x) for x in rng.integers(0, 1 << 40, 4)]
    _install(acc, st)
    adv, adv_g, adv_p = _adversarial(oracle, rng, cfg, st, n_adv)
    fr = list(frames) + adv + list(extra)
    gr = list(range(len(frames))) + adv_g + [int(rng.integers(0, G)) for _ in extra]
    pe = [int(rng.integers(0, cfg.n)) for _ in frames] + adv_p + [0] * len(extra)
    order = rng.permutation(len(fr))
    fr, gr, pe = [fr[i] for i in order], [gr[i] for i in order], [pe[i] for i in order]
    want, got = _run_and_check(ctx, acc, cfg, st, fr, gr, pe, rng, want_status=0)
    real = [k for k, i in enumerate(order) if i < len(frames)]
    assert all(want["verdict"][k] == ACC for k in real)
    _check_reply_parse(ctx, acc, cfg, want, got, gr, st)
    acc.close()
    return want


def _run_matrix(ctx, oracle, cfg_args, seed, variants=(2, 1, 3), force_pack=False, mes=None):
    protocol, n, d, T = cfg_args
    rng = np.random.default_rng(seed)
    mes = _mes(n) if mes is None else mes
    lens = _lens(rng, d)
    cfg0 = Cfg(protocol, n, 0, d, T, *variants)
    tables = _tables(oracle, rng, cfg0, mes)
    leader = _engine_takes(protocol, n, d, T) and not force_pack
    store = None if leader else _Store(oracle, rng, cfg0, lens)
    for me in mes:
        cfg = Cfg(protocol, n, me, d, T, *variants)
        if leader:
            frames, base, _, _ = _leader_frames(ctx, oracle, rng, protocol, n, T, d, False, me, lens.copy(),
                                                tables if cfg.cw else None)
        else:
            G = len(lens)
            base = rng.integers(0, 1 << 40, G).astype(np.uint64)
            slots = base + rng.integers(0, 64, G).astype(np.uint64)
            bals = rng.integers(1 << 20, 1 << 40, G).astype(np.uint64)
            pol = rng.integers(0, len(tables), G).astype(np.uint8)
            frames = _packed_frames(ctx, oracle, cfg, store, tables, pol, slots, bals, me)
        extra = _other_variant_frames(cfg) if variants != (2, 1, 3) else ()
        _matrix_cell(ctx, oracle, cfg, rng, frames, base, extra=extra)


@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,d,T", MATRIX)
def test_acceptor_matrix(ctx, oracle, protocol, n, d, T):
    _run_matrix(ctx, oracle, (protocol, n, d, T), seed=1000 * n + 37 * T + d + (protocol == "crossword"))


# ---------------------------------------------------------------------------------------------
# B: variant widths
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("av,wv,rv", VARIANT_SETTINGS)
@pytest.mark.parametrize("protocol", ["rspaxos", "crossword"])
def test_acceptor_variant_widths(ctx, oracle, protocol, av, wv, rv):
    code = ("rspaxos", 7, 4, 7) if protocol == "rspaxos" else ("crossword", 6, 4, 12)
    _run_matrix(ctx, oracle, code, seed=av % 1009 + wv % 997 + rv % 991, variants=(av, wv, rv), force_pack=True, mes=[code[1] // 2])


# ---------------------------------------------------------------------------------------------
# C: the widest reply cell and the data_len bound
# ---------------------------------------------------------------------------------------------
def _empty_accept(cfg, slot, ballot, dlen, rows):
    """a Crossword Accept that carries no shard (T Nones): tiny whatever data_len says"""
    body = b"\x00" + _vput(cfg.av) + _vput(slot) + _vput(ballot) + bytes([cfg.d, cfg.T - cfg.d]) + _vput(dlen)
    body += _vput(-(-dlen // cfg.d)) + _vput(cfg.T) + b"\x00" * cfg.T + b"\x00"
    body += _vput(len(rows)) + b"".join(_vput(cfg.T) + _vput(1) + _vput(r) for r in rows)
    return len(body).to_bytes(8, "big") + body


WIDE = Cfg("crossword", 3, 1, 1, 32, av=65536, wv=U32MAX, rv=U32MAX)
WIDE_ROWS = [0x0000ffff, 0xffffffff, 0xffff0000]


def test_model_widest_frames(oracle):
    """the model's decoder agrees with the oracle's on population 32 / T = 32 / wide-variant frames and on a frame that
    holds no shard at data_len 2^32 - 1; the widest reply the acceptor writes is 42 bytes"""
    slot, bal = (1 << 40) + 5, 1 << 33
    fr = _empty_accept(WIDE, slot, bal, U32MAX, WIDE_ROWS)
    f, o = _decode(fr, WIDE), oracle.decode_accept(fr, 0, True)
    assert o is not None and o["variant"] == WIDE.av and o["shards"] == [None] * 32
    assert (f["slot"], f["ballot"], f["dlen"], f["L"], f["held"], f["asg"]) == (slot, bal, U32MAX, U32MAX, 0, WIDE_ROWS)
    assert (o["slot"], o["ballot"], o["data_len"], o["shard_len"], o["assignment"]) == (slot, bal, U32MAX, U32MAX, WIDE_ROWS)
    assert _decode(_empty_accept(WIDE, slot, bal, 1 << 32, WIDE_ROWS), WIDE) == MALFORMED
    st = State(1)
    st.base = [slot - 3]
    r = _stream(WIDE, st, [fr], [0], [2], 1 << 20, 1 << 20)
    assert r["verdict"] == [ACC] and len(r["replies"][0]) == 42
    assert r["replies"][0] == oracle.frame_accept_reply(U32MAX, slot, bal, True, 1 << 37)
    assert oracle.parse_accept_reply(r["replies"][0], U32MAX, True) == (42, slot, bal, 1 << 37, U32MAX)
    # population 32, T = 32, every row full, every shard held, wide variants
    cfg = Cfg("crossword", 32, 31, 5, 32, av=U32MAX, wv=0, rv=65535)
    shards = [bytes([j]) * 3 for j in range(32)]
    fr = oracle.frame_accept(cfg.av, U64MAX, U64MAX - 1, 5, 27, 15, shards, [U32MAX] * 32, 32)
    f, o = _decode(fr, cfg), oracle.decode_accept(fr, 0, True)
    assert f["held"] == U32MAX and f["shards"] == o["shards"] == shards and f["asg"] == o["assignment"] == [U32MAX] * 32
    assert (f["slot"], f["ballot"], o["variant"]) == (U64MAX, U64MAX - 1, U32MAX)
    # the same frame spelled with every u64 varint in its 9-byte form
    from tests.test_acceptor import _acc_wide
    fw = _acc_wide(7, 9, 0x80000001, 40, 5, 27, [U32MAX] * 32, 32, av=U32MAX)
    f, o = _decode(fw, cfg), oracle.decode_accept(fw, 0, True)
    assert f["held"] == 0x80000001 and f["shards"] == o["shards"] and f["asg"] == o["assignment"]


@pytest.mark.gpu
def test_acceptor_widest_reply_and_data_len_bound(ctx, oracle):
    cfg = WIDE
    slot, bal = (1 << 40) + 5, 1 << 33
    rng = np.random.default_rng(42)
    acc = _acceptor(ctx, cfg, 2)
    st = State(2)
    st.base = [slot - 3, 0]
    _install(acc, st)
    frames = [_empty_accept(cfg, slot, bal, U32MAX, WIDE_ROWS), _empty_accept(cfg, slot + 1, bal, 1 << 32, WIDE_ROWS),
              _empty_accept(cfg, 3, 1, 0, [0, 0, 0])]
    want, got = _run_and_check(ctx, acc, cfg, st, frames, [0, 0, 1], [1, 2, 0], rng, want_status=0)
    assert want["verdict"] == [ACC, MALFORMED, ACC]
    assert int(got["reply_len"][0]) == 42 <= acc.REPLY_CELL
    assert got["replies"][0][:42].tobytes() == oracle.frame_accept_reply(U32MAX, slot, bal, True, 1 << 37)
    _check_reply_parse(ctx, acc, cfg, want, got, [0, 0, 1], st)
    acc.close()


# ---------------------------------------------------------------------------------------------
# D: batch sizes, scan tiles and grid caps
# ---------------------------------------------------------------------------------------------
def _copy_cap(ctx):
    return ctx.sm_count * 64 * 8          # launch_grid: 64 CTAs per SM; the copy kernel runs 8 warps (frames) per CTA


def _thread_cap(ctx):
    return ctx.sm_count * 64 * 256        # header, ballot, place and advance kernels: a thread per item


def _cheap_frames(oracle, rng, cfg, st, n):
    """n frames over st's groups: small, mostly inside the window, duplicate slots, ballots that rise with noise"""
    G = len(st.base)
    g = rng.integers(0, G, n)
    slot = np.array(st.base, dtype=np.int64)[g] + rng.integers(-2, 70, n)
    bal = np.arange(n) // 64 + rng.integers(0, 4, n) + 1
    held = rng.integers(1, 1 << cfg.T, n)
    dlen = rng.choice([1, 3, 17, 300], n)
    frames = [_oracle_accept(oracle, cfg.av, max(int(s), 0), int(b), cfg.d, cfg.T - cfg.d, int(dl),
                             [bytes([(i + j) & 255]) * (-(-int(dl) // cfg.d)) if (int(h) >> j) & 1 else None for j in range(cfg.T)],
                             None, cfg.T)
              for i, (s, b, h, dl) in enumerate(zip(slot, bal, held, dlen))]
    return frames, [int(x) for x in g], [int(x) % cfg.n for x in rng.integers(0, 256, n)]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2047, 2048, 2049, 4097, "copy_cap+1000"])
def test_acceptor_batch_sizes(ctx, oracle, n):
    if n == "copy_cap+1000":
        n = _copy_cap(ctx) + 1000
    cfg = Cfg("rspaxos", 3, 1, 2, 3)
    rng = np.random.default_rng(n)
    G = max(n // 40, 1)
    acc = _acceptor(ctx, cfg, G)
    st = State(G)
    st.base = [int(x) for x in rng.integers(0, 1 << 20, G)]
    _install(acc, st)
    frames, groups, peers = _cheap_frames(oracle, rng, cfg, st, n)
    want, _ = _run_and_check(ctx, acc, cfg, st, frames, groups, peers, rng, want_status=0)
    v = want["verdict"]
    assert v.count(ACC) > n // 4 and v.count(_lib.SS_ACCEPT_VERDICT_STALE_BALLOT) > 0
    acc.close()


@pytest.mark.gpu
def test_acceptor_past_the_header_grid_cap(ctx):
    """header-kernel cap + 1000 identical-length frames (RSPaxos, population 1, d = T = 1, 1-byte payloads, one ballot,
    3-byte slot varints): every frame is accepted, so offsets, records, replies and state follow from i in numpy"""
    N = _thread_cap(ctx) + 1000
    G = 1 << 16
    bal, base = 7, 1000
    acc = _acceptor(ctx, Cfg("rspaxos", 1, 0, 1, 1), G)
    i = np.arange(N, dtype=np.int64)
    g = (i % G).astype(np.uint32)
    slot = base + (i // G) % 64                                 # 1000..1063: (group, slot) unique, one varint width
    payload = ((i * 7 + 3) & 255).astype(np.uint8)
    peer = (i % 251).astype(np.uint8)
    # body: 00 02 | slot: fb lo hi | ballot | d p | data_len shard_len count | Some len byte | None
    F = 23
    fr = np.zeros((N, F), dtype=np.uint8)
    fr[:, 7] = F - 8
    fr[:, 8:10] = [0, 2]
    fr[:, 10] = 251
    fr[:, 11] = slot & 255
    fr[:, 12] = slot >> 8
    fr[:, 13:21] = [bal, 1, 0, 1, 1, 1, 1, 1]
    fr[:, 21] = payload
    fr[:, 22] = 0
    assert _decode(fr[0].tobytes(), Cfg("rspaxos", 1, 0, 1, 1))["L"] == 1
    assert fr[0].tobytes() == pyoracle.frame_accept(2, int(slot[0]), bal, 1, 0, 1, [bytes([payload[0]])])
    buf = np.concatenate([np.full(1, 0xEE, np.uint8), fr.reshape(-1), np.full(16, 0xEE, np.uint8)])
    offs = (1 + F * i).astype(np.uint64)
    st = State(G)
    st.base = [base] * G
    _install(acc, st)
    rng = np.random.default_rng(3)
    s_can = rng.integers(0, 256, 32 * N + 64, dtype=np.uint8)
    w_can = rng.integers(0, 256, 32 * N + 64, dtype=np.uint8)
    store, wal = _t(s_can), _t(w_can)
    out = acc.accept(_t(buf), _t(offs), _t(g), _t(peer), store, wal, 32 * N, 32 * N)
    assert ctx.device_status() == 0
    got = {k: v.cpu().numpy() for k, v in out.items()}
    assert (got["verdict"].view(np.uint32) == ACC).all()
    assert (got["store_off"].view(np.uint64) == 32 * i).all() and (got["wal_off"].view(np.uint64) == 32 * i).all()
    tail = F - 10                                               # the frame from `slot` on
    wl = 8 + 1 + tail
    assert (got["wal_len"] == wl).all() and list(got["totals"]) == [32 * N, 32 * N]
    ws = s_can.copy()
    ws[:32 * N].reshape(N, 32)[:, 0] = payload
    ws[:32 * N].reshape(N, 32)[:, 1:16] = 0
    assert np.array_equal(store.cpu().numpy(), ws)
    ww = w_can.copy()
    rec = np.zeros((N, wl), dtype=np.uint8)
    rec[:, 7] = wl - 8
    rec[:, 8] = 1
    rec[:, 9:] = fr[:, 10:]
    ww[:32 * N].reshape(N, 32)[:, :wl] = rec
    assert np.array_equal(wal.cpu().numpy(), ww)
    cell = np.zeros((N, 48), dtype=np.uint8)
    cell[:, 7] = 6
    cell[:, 9], cell[:, 10], cell[:, 11], cell[:, 12], cell[:, 13] = 3, 251, slot & 255, slot >> 8, bal
    assert cell[0, :14].tobytes() == pyoracle.frame_accept_reply(3, int(slot[0]), bal)
    assert np.array_equal(got["replies"], cell) and (got["reply_len"] == 14).all()
    assert np.array_equal(got["reply_dst"], peer)
    # state: every (group, slot) was named once
    torch.cuda.synchronize()
    at = g.astype(np.int64) * 64 + (slot & 63)
    ib = acc.inst_bal.cpu().numpy().view(np.uint64)
    assert (ib[at] == bal).all() and int(np.count_nonzero(ib)) == N
    assert (acc.source.cpu().numpy()[at] == peer).all()
    assert (acc.held.cpu().numpy()[at] == 1).all() and (acc.data_len.cpu().numpy()[at] == 1).all()
    assert (acc.shard_addr.cpu().numpy().view(np.uint64)[at] == np.uint64(store.data_ptr()) + (32 * i).astype(np.uint64)).all()
    cnt = np.bincount(g, minlength=G)                          # group g holds slots base .. base + cnt - 1
    r = base & 63
    ring = {c: (((1 << c) - 1) << r | ((1 << c) - 1) >> (64 - r)) & U64MAX for c in {int(x) for x in cnt}}
    want_acc = np.array([ring[int(c)] for c in cnt], dtype=np.uint64)
    assert np.array_equal(acc.accepting.cpu().numpy().view(np.uint64), want_acc)
    assert (acc.bal_max_seen.cpu().numpy() == bal).all()
    acc.close()


@pytest.mark.gpu
def test_acceptor_advance_past_its_grid_cap(ctx):
    """advance over advance-kernel cap + 1000 groups (about 3.6 GB of RSPaxos state): upto below the base, at it, at
    base + 1, 63, 64, 65 and at 2^64 - 1, group by group"""
    G = _thread_cap(ctx) + 1000
    acc = _acceptor(ctx, Cfg("rspaxos", 3, 0, 2, 3), G)
    rng = np.random.default_rng(11)
    base = rng.integers(5, 1 << 62, G, dtype=np.uint64)
    word = rng.integers(0, 1 << 63, G, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, G, dtype=np.uint64)
    acc.window_base.copy_(_t(base))
    acc.accepting.copy_(_t(word))
    rel = np.array([-5, 0, 1, 63, 64, 65, 0], dtype=np.int64)
    kind = np.arange(G) % 7
    upto = (base.astype(np.int64) + rel[kind]).astype(np.uint64)
    upto[kind == 6] = np.uint64(U64MAX)
    acc.advance(_t(upto))
    torch.cuda.synchronize()
    k = np.where(upto <= base, np.uint64(0), np.minimum(upto - base, np.uint64(64)))
    assert np.array_equal(acc.window_base.cpu().numpy().view(np.uint64), base + k)
    # ring positions kept: window bits k.. rotated to the ring by base & 63
    keep_w = np.where(k == 64, np.uint64(0), np.left_shift(np.uint64(U64MAX), np.minimum(k, np.uint64(63))))
    r = base & np.uint64(63)
    keep = np.left_shift(keep_w, r) | np.right_shift(keep_w, (np.uint64(64) - r) & np.uint64(63))
    assert np.array_equal(acc.accepting.cpu().numpy().view(np.uint64), word & keep)
    acc.close()


# ---------------------------------------------------------------------------------------------
# E: sort keys around powers of two
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 2, 3, 4, 5, 255, 256, 257, 65535, 65536, 65537])
def test_acceptor_sort_keys(ctx, oracle, G):
    """frames to every group, interleaved, several to a few groups with falling ballots, and frames naming G, G + 1 and
    2^32 - 1 (malformed): a key width one bit short merges groups and breaks their ballot order"""
    cfg = Cfg("rspaxos", 1, 0, 1, 1)
    rng = np.random.default_rng(G)
    acc = _acceptor(ctx, cfg, G)
    st = State(G)
    st.base = [int(x) for x in rng.integers(0, 1 << 30, G)]
    _install(acc, st)
    hot = sorted({0, G - 1, G // 2, min(G - 1, 32768), min(G - 1, 128)})
    groups = list(rng.permutation(G)) + [int(h) for h in hot for _ in range(6)] + [G, G + 1, U32MAX]
    rng.shuffle(groups)
    frames = []
    for k, g in enumerate(groups):
        b = st.base[g] if g < G else 0
        frames.append(_oracle_accept(oracle, 2, b + int(rng.integers(0, 4)), int(rng.integers(1, 9)), 1, 0, 1, [bytes([k & 255])], None, 1))
    want, _ = _run_and_check(ctx, acc, cfg, st, frames, [int(x) for x in groups], [0] * len(groups), rng, want_status=0)
    v = want["verdict"]
    assert [v[i] for i, g in enumerate(groups) if g >= G] == [MALFORMED] * 3
    assert v.count(_lib.SS_ACCEPT_VERDICT_STALE_BALLOT) > 0
    acc.close()


# ---------------------------------------------------------------------------------------------
# F: one acceptor across calls
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_acceptor_across_calls(ctx, oracle):
    """scratch grows (3 -> 5000 -> copy cap + 1000), is reused at 1 and 17, state carried through the model"""
    cfg = Cfg("crossword", 4, 2, 3, 8)
    rng = np.random.default_rng(77)
    G = 3001
    acc = _acceptor(ctx, cfg, G)
    st = State(G)
    st.base = [int(x) for x in rng.integers(0, 1 << 36, G)]
    _install(acc, st)
    for call, n in enumerate([3, 5000, 1, _copy_cap(ctx) + 1000, 17]):
        frames, groups, peers = _adversarial(oracle, rng, cfg, st, n)
        _run_and_check(ctx, acc, cfg, st, frames, groups, peers, rng, want_status=0)
        if call in (1, 3):
            upto = [b + int(rng.integers(0, 70)) for b in st.base]
            acc.advance(_t(np.array(upto, dtype=np.uint64)))
            _advance(st, upto)
    _check_state(acc, cfg, st, 0)
    acc.close()


# ---------------------------------------------------------------------------------------------
# G: one hot group
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_acceptor_one_hot_group(ctx, oracle):
    """20k frames of one group over its 64 slots (many per slot, ballots random but rising), and a few hundred others"""
    cfg = Cfg("crossword", 5, 4, 3, 5)
    rng = np.random.default_rng(5)
    G = 97
    acc = _acceptor(ctx, cfg, G)
    st = State(G)
    st.base = [int(x) for x in rng.integers(0, 1 << 40, G)]
    st.bmax = [3] * G
    _install(acc, st)
    n_hot, n_cold = 20000, 400
    groups = np.where(rng.random(n_hot + n_cold) < n_hot / (n_hot + n_cold), 17, rng.integers(0, G, n_hot + n_cold))
    rows = [[int(x) for x in pyoracle.cw_brr_assignment(5, 5, 2)], [0b11111, 0, 0b1, 0b10, 0b100]]
    frames, peers = [], []
    for k, g in enumerate(groups):
        slot = st.base[g] + int(rng.integers(0, 64))
        bal = k // 20 + int(rng.integers(0, 3))
        held = int(rng.integers(0, 32))
        dl = int(rng.choice([1, 9, 100]))
        L = -(-dl // 3)
        frames.append(_oracle_accept(oracle, 2, slot, bal, 3, 2, dl, [bytes([k & 255]) * L if (held >> j) & 1 else None for j in range(5)],
                                     rows[k & 1], 5))
        peers.append(int(rng.integers(0, 5)))
    want, _ = _run_and_check(ctx, acc, cfg, st, frames, [int(x) for x in groups], peers, rng, want_status=0)
    v = [want["verdict"][i] for i in range(len(groups)) if groups[i] == 17]
    assert v.count(ACC) > 1000 and v.count(_lib.SS_ACCEPT_VERDICT_STALE_BALLOT) > 1000
    assert len(st.inst[17]) == 64
    acc.close()


# ---------------------------------------------------------------------------------------------
# I: a non-blocking context stream while torch's default stream is busy
# ---------------------------------------------------------------------------------------------
SLEEP_CYCLES = 1_000_000_000          # about 0.5 s at the H100's clocks


def _pinned(ctx, arr):
    lib = ctx.lib
    p = C.c_void_p()
    assert lib.ss_host_alloc(ctx.h, arr.nbytes, C.byref(p)) == _lib.SS_OK
    C.memmove(p.value, arr.ctypes.data, arr.nbytes)
    return p


@pytest.mark.gpu
def test_acceptor_on_a_non_blocking_stream(oracle):
    """Creation zeroes the acceptor's arrays on the context's stream: with torch's default stream busy, the caller's
    window_base and the first accept on a non-blocking context stream are kept"""
    from summerset_b200.api import Context
    from summerset_b200.engine import Acceptor
    cfg = Cfg("crossword", 5, 1, 3, 10)
    rng = np.random.default_rng(8)
    G = 37
    st = State(G)
    st.base = [int(x) for x in rng.integers(1, 1 << 40, G)]
    frames, groups, peers = _adversarial(oracle, rng, cfg, st, 300)
    buf, offs = _buffer(rng, frames)
    mv = memoryview(buf.tobytes())
    want = _stream(cfg, st, [mv[int(o):] for o in offs], groups, peers, 1 << 40, 1 << 40)
    n = len(frames)
    s_tot, w_tot = want["totals"]
    d_buf, d_off, d_grp, d_peer = _t(buf), _t(offs), _t(np.array(groups, np.uint32)), _t(np.array(peers, np.uint8))
    store, wal = torch.zeros(s_tot + 64, dtype=torch.uint8, device=DEV), torch.zeros(w_tot + 64, dtype=torch.uint8, device=DEV)
    o = {k: torch.zeros(n * w, dtype=torch.uint8, device=DEV) for k, w in (("store_off", 8), ("wal_off", 8), ("wal_len", 4),
                                                                           ("replies", 48), ("reply_len", 4), ("reply_dst", 1),
                                                                           ("verdict", 4))}
    totals = torch.zeros(2, dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    ctx = Context(0, own_stream=True)
    base_arr = np.array(st.base, dtype=np.uint64)               # _stream moves no base
    host_base = _pinned(ctx, base_arr)
    torch.cuda._sleep(SLEEP_CYCLES)
    acc = Acceptor(ctx, cfg.protocol, G, cfg.n, cfg.me, cfg.d, cfg.T)
    lib = ctx.lib
    assert lib.ss_copy_h2d(ctx.h, acc.view.window_base, host_base, base_arr.nbytes) == _lib.SS_OK
    p = lambda x: x.data_ptr()
    assert lib.ss_acceptor_accept(acc.h, p(d_buf), d_buf.numel(), p(d_off), p(d_grp), p(d_peer), n, p(store), s_tot, p(o["store_off"]),
                                  p(wal), w_tot, p(o["wal_off"]), p(o["wal_len"]), p(o["replies"]), p(o["reply_len"]),
                                  p(o["reply_dst"]), p(o["verdict"]), p(totals)) == _lib.SS_OK
    assert lib.ss_ctx_sync(ctx.h) == _lib.SS_OK
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in o.items()}
    assert [int(x) for x in got["verdict"].view(np.uint32)] == want["verdict"]
    assert [int(x) for x in got["store_off"].view(np.uint64)] == want["store_off"]
    assert [int(x) for x in got["wal_off"].view(np.uint64)] == want["wal_off"]
    assert [int(x) for x in got["wal_len"].view(np.uint32)] == want["wal_len"]
    cells = got["replies"].reshape(n, 48)
    for i in range(n):
        r = want["replies"][i] or b""
        assert cells[i, :len(r)].tobytes() == r and not cells[i, len(r):].any(), i
    w = wal.cpu().numpy()
    for i in range(n):
        if want["verdict"][i] == ACC:
            assert w[want["wal_off"][i]:want["wal_off"][i] + want["wal_len"][i]].tobytes() == want["records"][i], i
    assert ctx.device_status() == 0
    _check_state(acc, cfg, st, p(store))
    assert lib.ss_host_free(ctx.h, host_base) == _lib.SS_OK
    acc.close()
    ctx.close()


@pytest.mark.gpu
def test_engine_on_a_non_blocking_stream():
    """the engine's arrays are zeroed on the context's stream: prepared ballots written right after creation stay"""
    from summerset_b200.api import Context
    from summerset_b200.engine import LeaderEngine
    G = 4096
    bal = np.random.default_rng(2).integers(1, 1 << 50, G).astype(np.uint64)
    d_bal = _t(bal)
    torch.cuda.synchronize()
    ctx = Context(0, own_stream=True)
    torch.cuda._sleep(SLEEP_CYCLES)
    eng = LeaderEngine(ctx, "multipaxos", G, 5)
    eng.set_prepared_ballots(d_bal)
    ctx.sync()
    torch.cuda.synchronize()
    assert np.array_equal(eng.bal_prepared.cpu().numpy().view(np.uint64), bal)
    eng.close()
    ctx.close()


@pytest.mark.gpu
def test_acceptor_matrix_cell_on_own_stream(oracle):
    """one matrix cell on a context with its own non-blocking stream, torch's ops ordered on that stream"""
    from summerset_b200.api import Context
    c = Context(0, own_stream=True)
    s = torch.cuda.ExternalStream(c.lib.ss_ctx_stream(c.h), device=DEV)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        _run_matrix(c, oracle, ("crossword", 7, 7, 14), seed=14)
    c.sync()
    c.close()


# ---------------------------------------------------------------------------------------------
# J: the AcceptReply parser's frame bounds
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_accept_reply_parse_bounds(ctx, oracle):
    """frame_off at buf_len - 9 .. buf_len + 1 and 2^64 - 8 .. 2^64 - 1, groups at and past n_groups.  buf sits 16 bytes
    into its allocation behind guard bytes that spell a well-formed reply for a parse that starts before buf, so a
    wrapped bound reads inside the allocation and shows up as a wrong record, not a fault"""
    rv, G = 3, 4
    base = np.array([100, 0, 1 << 40, 7], dtype=np.uint64)
    frames = [oracle.frame_accept_reply(rv, 100 + k, 9 + k) for k in range(3)] + [oracle.frame_accept_reply(5, 1, 1)]
    frames += [oracle.frame_accept_reply(rv, 7, 1 << 35)]
    body = b"".join(frames) + (1).to_bytes(8, "big") + b"\x05"           # ends with a 1-byte LeaseMsg-like frame
    blen = len(body)
    guard = (0).to_bytes(8, "big") + (6).to_bytes(8, "big")              # a frame at buf - 8 would read body[0:6]
    raw = np.frombuffer(guard + body + b"\x00" * 16, dtype=np.uint8).copy()
    buf = _t(raw)[16:16 + blen]
    starts = np.cumsum([0] + [len(f) for f in frames])[:-1]
    offs = [int(x) for x in starts] + list(range(blen - 9, blen + 2)) + [(1 << 64) - k for k in range(8, 0, -1)]
    grp = [0, 0, 0, 0, 3] + [0] * (len(offs) - 5)
    offs += [0, int(starts[4]), int(starts[4])]
    grp += [G, G + 1, U32MAX]
    rg, rs_, rp, rb, rk = ctx.accept_reply_parse(buf, _t(np.array(offs, dtype=np.uint64)), _t(np.array(grp, dtype=np.uint32)),
                                                 _t(np.arange(len(offs), dtype=np.uint8)), _t(base), rv, False)
    rs_, rb, rk, rp = rs_.cpu().numpy(), rb.cpu().numpy().view(np.uint64), rk.cpu().numpy().view(np.uint32), rp.cpu().numpy()
    assert (rg.cpu().numpy().view(np.uint32) == np.array(grp, dtype=np.uint32)).all() and (rp == np.arange(len(offs))).all()
    for i, (off, g) in enumerate(zip(offs, grp)):
        if off > blen or blen - off < 8:
            want = (MALFORMED, 0xFF, 0)
        else:
            n, slot, bal, _, kind = oracle.parse_accept_reply(body[off:], rv, False)
            if n == -1:
                want = (MALFORMED, 0xFF, 0)
            elif n == -2:
                want = (kind, 0xFF, 0)
            else:
                b = int(base[g]) if g < G else None
                want = (rv, slot - b if b is not None and b <= slot < b + 64 else 0xFF, bal)
        assert (int(rk[i]), int(rs_[i]), int(rb[i])) == want, (i, off, g)
    assert [int(x) for x in rk[:5]] == [rv, rv, rv, 5, rv] and [int(x) for x in rs_[:5]] == [0, 1, 2, 0xFF, 0]


# ---------------------------------------------------------------------------------------------
# CPU: configuration edges
# ---------------------------------------------------------------------------------------------
def test_acceptor_create_config_edges():
    lib = _lib.load()
    h = C.c_void_p()
    P = _lib.SS_PROTO_CROSSWORD
    for cfg, G in ((_lib.AcceptorConfig(P, 32, 32, 3, 32, 2, 1, 3), 16), (_lib.AcceptorConfig(P, 5, 1, 3, 33, 2, 1, 3), 16),
                   (_lib.AcceptorConfig(_lib.SS_PROTO_RSPAXOS, 5, 1, 3, 5, 2, 1, 3), 1 << 32)):
        assert lib.ss_acceptor_create(None, C.byref(cfg), G, C.byref(h)) == _lib.SS_ERR_INVALID_ARG and not h


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_acceptor_create_config_edges_pass_the_checks():
    lib = _lib.load()
    h = C.c_void_p()
    for cfg, G in ((_lib.AcceptorConfig(_lib.SS_PROTO_CROSSWORD, 32, 31, 1, 32, U32MAX, 0, 65536), (1 << 32) - 1),
                   (_lib.AcceptorConfig(_lib.SS_PROTO_RSPAXOS, 1, 0, 32, 32, 2, 1, 3), 1)):
        assert lib.ss_acceptor_create(None, C.byref(cfg), G, C.byref(h)) == _lib.SS_ERR_NO_DEVICE and not h
