"""The follower side of the RSPaxos / Crossword accept path (ss_acceptor_*, summerset_b200/csrc/acceptor.cu).

`_stream` below restates handle_msg_accept per message (rspaxos/messages.rs:329-392, crossword/messages.rs:403-470) with
check_leader's bal_max_seen update (rspaxos/leadership.rs:11-17), in frame order, over the acceptor's state and window
rule; it returns the verdicts, the final state and the records and replies a host would emit.  Frames are decoded by
hand here and cross-checked with the oracle's ssor_decode_accept; records and replies are built from the oracle's
encoders.  The GPU tests drive the C ABI and compare every byte and every state word with it.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pyoracle
from summerset_b200 import _lib

DEV = "cuda:0"
ACC, STALE_SLOT, STALE_BAL, BEYOND, STORE_FULL_V, WAL_FULL_V, MALFORMED = (
    _lib.SS_ACCEPT_VERDICT_ACCEPTED, _lib.SS_ACCEPT_VERDICT_STALE_SLOT, _lib.SS_ACCEPT_VERDICT_STALE_BALLOT,
    _lib.SS_ACCEPT_VERDICT_BEYOND_WINDOW, _lib.SS_ACCEPT_VERDICT_STORE_FULL, _lib.SS_ACCEPT_VERDICT_WAL_FULL,
    _lib.SS_FRAME_KIND_MALFORMED)
FRAME_OVERFLOW, STORE_FULL = 4, 16
U64MAX = (1 << 64) - 1


# ---------------------------------------------------------------------------------------------
# the per-message model
# ---------------------------------------------------------------------------------------------
def _vput(v):
    if v < 251:
        return bytes([v])
    for nb, tag in ((2, 251), (4, 252), (8, 253)):
        if v < 1 << (8 * nb):
            return bytes([tag]) + v.to_bytes(nb, "little")


def _vget(b, n):
    if n >= len(b):
        return None
    t = b[n]
    if t < 251:
        return t, n + 1
    nb = {251: 2, 252: 4, 253: 8}.get(t)
    if nb is None or n + 1 + nb > len(b):
        return None
    return int.from_bytes(b[n + 1:n + 1 + nb], "little"), n + 1 + nb


class Cfg:
    def __init__(self, protocol, n, me, d, T, av=2, wv=1, rv=3):
        self.cw = protocol == "crossword"
        self.protocol, self.n, self.me, self.d, self.T, self.av, self.wv, self.rv = protocol, n, me, d, T, av, wv, rv


def _decode(frame, cfg):
    """-> dict of the Accept, or the verdict of a frame that is not one this acceptor takes"""
    if len(frame) < 8:
        return MALFORMED
    ln = int.from_bytes(frame[:8], "big")
    if ln > len(frame) - 8:
        return MALFORMED
    b = frame[8:8 + ln]
    r = _vget(b, 0)
    if r is None:
        return MALFORMED
    if r[0] != 0:
        return 0x80000000 | r[0] if r[0] < 1 << 16 else MALFORMED
    r = _vget(b, r[1])
    if r is None:
        return MALFORMED
    if r[0] != cfg.av:
        return r[0] if r[0] < 1 << 16 else MALFORMED
    slot_at = 8 + r[1]
    f = {}
    n = r[1]
    for k in ("slot", "ballot"):
        r = _vget(b, n)
        if r is None:
            return MALFORMED
        f[k], n = r
    if len(b) - n < 2 or b[n] != cfg.d or b[n + 1] != cfg.T - cfg.d:
        return MALFORMED
    n += 2
    vals = []
    for _ in range(3):
        r = _vget(b, n)
        if r is None:
            return MALFORMED
        vals.append(r[0])
        n = r[1]
    dl, sl, cnt = vals
    if dl >= 1 << 32 or cnt != cfg.T or sl != -(-dl // cfg.d):
        return MALFORMED
    held, shards = 0, []
    for j in range(cfg.T):
        if n >= len(b):
            return MALFORMED
        tag = b[n]
        n += 1
        if tag == 0:
            shards.append(None)
            continue
        if tag != 1:
            return MALFORMED
        r = _vget(b, n)
        if r is None or r[0] != sl or len(b) - r[1] < sl:
            return MALFORMED
        n = r[1]
        shards.append(bytes(b[n:n + sl]))
        held |= 1 << j
        n += sl
    if n >= len(b) or b[n] != 0:
        return MALFORMED
    n += 1
    asg = None
    if cfg.cw:
        r = _vget(b, n)
        if r is None or r[0] != cfg.n:
            return MALFORMED
        n, asg = r[1], []
        for _ in range(cfg.n):
            row = []
            for _ in range(3):
                r = _vget(b, n)
                if r is None:
                    return MALFORMED
                row.append(r[0])
                n = r[1]
            if row[0] != cfg.T or row[1] != 1 or row[2] >> cfg.T:
                return MALFORMED
            asg.append(row[2])
    if n != len(b):
        return MALFORMED
    f.update(dlen=dl, L=sl, held=held, shards=shards, asg=asg, slot_at=slot_at, end=8 + ln)
    return f


def _pitch(L):
    return (L + 31) // 32 * 32


def _wal_record(frame, f, cfg):
    body = _vput(cfg.wv) + bytes(frame[f["slot_at"]:f["end"]])
    return len(body).to_bytes(8, "big") + body


def _reply(cfg, slot, inst):
    body = _vput(0) + _vput(cfg.rv) + _vput(slot) + _vput(inst["bal"])
    if cfg.cw:
        body += _vput(bin(inst["asg"][cfg.me]).count("1") * (inst["dlen"] // cfg.d + 1)) + b"\x00"
    return len(body).to_bytes(8, "big") + body


class State:
    def __init__(self, G):
        self.base = [0] * G
        self.bmax = [0] * G
        self.inst = [dict() for _ in range(G)]       # slot -> dict(bal, src, held, dlen, asg, store_at)


def _stream(cfg, st, frames, groups, peers, store_cap, wal_cap):
    """One call, one message at a time in frame order, as handle_msg_accept meets them: verdicts, offsets, records and
    replies; st is updated in place.  `run` is check_leader's bal_max_seen as each frame reaches the ballot check; a frame
    that passes it but finds no room in the store or the WAL keeps its place in that order and changes nothing else
    (bal_max_seen at the end is the highest ACCEPTED ballot).  Replies are built once the whole batch is logged."""
    n = len(frames)
    G = len(st.base)
    verdict, dec = [None] * n, [None] * n
    store_off, wal_off, wal_len = [U64MAX] * n, [U64MAX] * n, [0] * n
    run = list(st.bmax)
    s_at = w_at = 0
    for i, (fr, g) in enumerate(zip(frames, groups)):
        if g >= G:                                    # a group this acceptor does not hold: malformed, whatever the frame
            verdict[i] = MALFORMED
            continue
        f = _decode(fr, cfg)
        if isinstance(f, int):
            verdict[i] = f
            continue
        dec[i] = f
        if f["slot"] < st.base[g]:                    # `slot < start_slot`: ignored
            verdict[i] = STALE_SLOT
            continue
        if f["slot"] >= st.base[g] + 64:              # beyond the window: re-submitted later
            verdict[i] = BEYOND
            continue
        if f["ballot"] < run[g]:                      # `ballot >= bal_max_seen` fails
            verdict[i] = STALE_BAL
            continue
        run[g] = f["ballot"]                          # check_leader
        sz = bin(f["held"]).count("1") * _pitch(f["L"])
        wl = 8 + len(_vput(cfg.wv)) + f["end"] - f["slot_at"]
        wz = (wl + 15) // 16 * 16
        so, wo = s_at, w_at
        s_at += sz
        w_at += wz
        if so + sz > store_cap:
            verdict[i] = STORE_FULL_V
            continue
        if wo + wz > wal_cap:
            verdict[i] = WAL_FULL_V
            continue
        verdict[i] = ACC
        store_off[i], wal_off[i], wal_len[i] = so, wo, wl
        st.bmax[g] = max(st.bmax[g], f["ballot"])
        # inst.bal, status, reqs_cw, assignment, replica_bk.source: the later frame of a slot overwrites
        st.inst[g][f["slot"]] = dict(bal=f["ballot"], src=peers[i], held=f["held"], dlen=f["dlen"], asg=f["asg"], store_at=so,
                                     fresh=True)
    records, replies, dst = [None] * n, [None] * n, [0xFF] * n
    for i in range(n):
        if verdict[i] == ACC:
            f, g = dec[i], groups[i]
            records[i] = _wal_record(frames[i], f, cfg)
            inst = st.inst[g][f["slot"]]
            replies[i] = _reply(cfg, f["slot"], inst)
            dst[i] = inst["src"]
    return dict(verdict=verdict, dec=dec, store_off=store_off, wal_off=wal_off, wal_len=wal_len, records=records, replies=replies,
                reply_dst=dst, totals=(s_at, w_at))


def _oracle_record(oracle, cfg, f):
    """WalEntry::AcceptData re-encoded from the decoded fields by the oracle's encoders; Crossword appends
    assignment: Vec<Bitmap> (crossword/mod.rs:288-293) after the oracle's RSPaxos-shaped record body.  The oracle
    writes the record variant as 1 (one byte): the body after it is kept, the variant is the acceptor's wal_variant."""
    rec = oracle.wal_accept_data(f["slot"], f["ballot"], cfg.d, cfg.T - cfg.d, f["dlen"], f["shards"])
    assert rec[8] == 1
    body = oracle.varint(cfg.wv) + rec[9:]
    if cfg.cw:
        body += oracle.varint(len(f["asg"])) + b"".join(oracle.bitmap_encode(cfg.T, a) for a in f["asg"])
    return len(body).to_bytes(8, "big") + body


def _oracle_frame(oracle, cfg, f):
    return oracle.frame_accept(cfg.av, f["slot"], f["ballot"], cfg.d, cfg.T - cfg.d, f["dlen"], f["shards"], f["asg"], cfg.T)


def _oracle_reply(oracle, cfg, slot, inst):
    size = bin(inst["asg"][cfg.me]).count("1") * (inst["dlen"] // cfg.d + 1) if cfg.cw else 0
    return oracle.frame_accept_reply(cfg.rv, slot, inst["bal"], cfg.cw, size)


def _advance(st, upto):
    for g, u in enumerate(upto):
        k = min(max(u - st.base[g], 0), 64)
        for s in [s for s in st.inst[g] if s < st.base[g] + k]:
            del st.inst[g][s]
        st.base[g] += k


# ---------------------------------------------------------------------------------------------
# CPU: the model on hand-written cases
# ---------------------------------------------------------------------------------------------
RS = Cfg("rspaxos", 5, 1, 3, 5)


def _acc(oracle, slot, ballot, held=0b00010, dlen=9, d=3, p=2, asg=None, T=5, av=2):
    L = -(-dlen // d)
    shards = [bytes([(slot + j) & 255]) * L if (held >> j) & 1 else None for j in range(d + p)]
    if not any(shards):
        shards[0] = b""
    return oracle.frame_accept(av, slot, ballot, d, p, dlen, shards, asg, T)


def _acc_wide(slot, ballot, held, dlen, d, p, asg, T, av=2):
    """an Accept whose every u64 varint uses the 9-byte form (tag 253): not minimal, but what the crate's decoder and
    the oracle's read as the same values"""
    w = lambda v: bytes([253]) + int(v).to_bytes(8, "little")
    L = -(-dlen // d)
    body = b"\x00" + _vput(av) + w(slot) + w(ballot) + bytes([d, p]) + w(dlen) + w(L) + w(d + p)
    for j in range(d + p):
        body += (b"\x01" + w(L) + bytes([(slot + 3 * j) & 255]) * L) if (held >> j) & 1 else b"\x00"
    body += b"\x00"
    if asg is not None:
        body += w(len(asg)) + b"".join(w(T) + w(1) + w(a) for a in asg)
    return len(body).to_bytes(8, "big") + body


def test_model_non_minimal_varints(oracle):
    """non-minimal varints decode to the same fields (the oracle agrees); the record keeps the frame's bytes"""
    cfg = Cfg("crossword", 5, 1, 3, 5)
    fr = _acc_wide(300, 7, 0b10110, 700, 3, 2, CW_ROWS, 5)
    f = _decode(fr, cfg)
    o = oracle.decode_accept(fr, 0, True)
    assert o is not None and (o["slot"], o["ballot"], o["data_len"], o["shards"], o["assignment"]) == \
        (f["slot"], f["ballot"], f["dlen"], f["shards"], f["asg"])
    st = State(1)
    st.base = [256]
    r = _stream(cfg, st, [fr], [0], [2], 1 << 20, 1 << 20)
    assert r["verdict"] == [ACC] and r["records"][0][9:] == fr[10:]
    assert oracle.decode_accept(r["records"][0], 1, True)["shards"] == f["shards"]


def test_model_ballot_order_in_one_group(oracle):
    st = State(2)
    st.bmax = [5, 0]
    frames = [_acc(oracle, 0, 7), _acc(oracle, 1, 6), _acc(oracle, 2, 9), _acc(oracle, 3, 8), _acc(oracle, 3, 100)]
    groups = [0, 0, 0, 0, 1]
    r = _stream(RS, st, frames, groups, [4, 4, 2, 4, 3], 1 << 20, 1 << 20)
    # 7 passes (>= 5) and raises to 7; 6 is stale; 9 passes; 8 is stale; group 1 is independent
    assert r["verdict"] == [ACC, STALE_BAL, ACC, STALE_BAL, ACC]
    assert st.bmax == [9, 100]
    assert sorted(st.inst[0]) == [0, 2] and st.inst[0][2]["src"] == 2
    assert r["store_off"] == [0, U64MAX, 32, U64MAX, 64]


def test_model_two_accepts_for_one_slot(oracle):
    st = State(1)
    frames = [_acc(oracle, 4, 3), _acc(oracle, 4, 3, held=0b00100), _acc(oracle, 4, 8, held=0b11000)]
    r = _stream(RS, st, frames, [0, 0, 0], [1, 2, 3], 1 << 20, 1 << 20)
    assert r["verdict"] == [ACC, ACC, ACC]
    inst = st.inst[0][4]
    assert inst["bal"] == 8 and inst["src"] == 3 and inst["held"] == 0b11000
    # every accepted frame has its own record; every reply carries the instance as the call left it
    assert len({bytes(x) for x in r["records"]}) == 3
    assert r["replies"] == [oracle.frame_accept_reply(3, 4, 8)] * 3 and r["reply_dst"] == [3, 3, 3]


def test_model_stale_slot_beyond_window_malformed(oracle):
    st = State(1)
    st.base = [100]
    good = _acc(oracle, 130, 1)
    frames = [_acc(oracle, 99, 50),            # stale slot carrying the highest ballot: must not raise bal_max_seen
              _acc(oracle, 164, 40),           # beyond the window: takes no part either
              good[:-1],                       # truncated
              _acc(oracle, 130, 1, d=2, p=3),  # another code
              oracle.frame_accept_reply(3, 130, 1),
              b"\x00" * 7 + b"\x01" + b"\x02",  # PeerMessage variant 2
              good]
    r = _stream(RS, st, frames, [0] * 7, [0] * 7, 1 << 20, 1 << 20)
    assert r["verdict"] == [STALE_SLOT, BEYOND, MALFORMED, MALFORMED, 3, 0x80000002, ACC]
    assert st.bmax == [1]


def test_model_shard_len_rule(oracle):
    # shard_len must be ceil(data_len / d); a frame that says otherwise is malformed
    cw = oracle.frame_accept(2, 0, 1, 3, 2, 9, [b"abc", None, None, None, None])
    assert _decode(cw, RS)["L"] == 3
    bad = oracle.frame_accept(2, 0, 1, 3, 2, 10, [b"abc", None, None, None, None])
    assert oracle.decode_accept(bad, 0) is not None and _decode(bad, RS) == MALFORMED


# hand-written bincode: Crossword RS(3,2), 5 replicas, me = 1, slot 300, ballot 7, data_len 6 (divisible by d: the
# reply's size is 2 shards * (6/3 + 1) = 6, where ceil would give 4)
CW_ROWS = [0b00011, 0b00110, 0b01100, 0b11000, 0b10001]
CW_BODY_TAIL = bytes([0xFB, 0x2C, 0x01, 0x07, 0x03, 0x02, 0x06, 0x02, 0x05, 0x00, 0x01, 0x02, 0xAA, 0xBB, 0x01, 0x02, 0xCC, 0xDD,
                      0x00, 0x00, 0x00, 0x05, 0x05, 0x01, 0x03, 0x05, 0x01, 0x06, 0x05, 0x01, 0x0C, 0x05, 0x01, 0x18, 0x05, 0x01,
                      0x11])
CW_FRAME = (len(CW_BODY_TAIL) + 2).to_bytes(8, "big") + b"\x00\x02" + CW_BODY_TAIL
CW_WAL = (len(CW_BODY_TAIL) + 1).to_bytes(8, "big") + b"\x01" + CW_BODY_TAIL
CW_REPLY = bytes([0, 0, 0, 0, 0, 0, 0, 8, 0x00, 0x03, 0xFB, 0x2C, 0x01, 0x07, 0x06, 0x00])


def test_crossword_accept_data_and_reply_bytes(oracle):
    cfg = Cfg("crossword", 5, 1, 3, 5)
    assert oracle.frame_accept(2, 300, 7, 3, 2, 6, [None, b"\xaa\xbb", b"\xcc\xdd", None, None], CW_ROWS, 5) == CW_FRAME
    st = State(1)
    st.base = [256]
    r = _stream(cfg, st, [CW_FRAME], [0], [0], 1 << 20, 1 << 20)
    assert r["verdict"] == [ACC] and r["records"][0] == CW_WAL and r["replies"][0] == CW_REPLY
    assert oracle.frame_accept_reply(3, 300, 7, True, 6) == CW_REPLY
    assert oracle.decode_accept(CW_WAL, 1, True)["assignment"] == CW_ROWS
    # the RSPaxos record is the oracle's AcceptData
    rs = _acc(oracle, 300, 7)
    r = _stream(RS, st, [rs], [0], [0], 1 << 20, 1 << 20)
    f = r["dec"][0]
    assert r["records"][0] == oracle.wal_accept_data(300, 7, 3, 2, 9, f["shards"])


def test_acceptor_symbols_and_refusals():
    lib = _lib.load()
    for name in ("ss_acceptor_create", "ss_acceptor_destroy", "ss_acceptor_view_get", "ss_acceptor_window_get",
                 "ss_acceptor_advance", "ss_acceptor_accept"):
        assert hasattr(lib, name)
    h = C.c_void_p()
    good = _lib.AcceptorConfig(_lib.SS_PROTO_RSPAXOS, 5, 1, 3, 5, 2, 1, 3)
    for bad in (_lib.AcceptorConfig(_lib.SS_PROTO_MULTIPAXOS, 5, 1, 3, 5, 2, 1, 3), _lib.AcceptorConfig(_lib.SS_PROTO_RAFT, 5, 1, 3, 5, 2, 1, 3),
                _lib.AcceptorConfig(_lib.SS_PROTO_RSPAXOS, 0, 0, 3, 5, 2, 1, 3), _lib.AcceptorConfig(_lib.SS_PROTO_RSPAXOS, 5, 5, 3, 5, 2, 1, 3),
                _lib.AcceptorConfig(_lib.SS_PROTO_CROSSWORD, 5, 1, 0, 5, 2, 1, 3), _lib.AcceptorConfig(_lib.SS_PROTO_CROSSWORD, 5, 1, 6, 5, 2, 1, 3),
                _lib.AcceptorConfig(_lib.SS_PROTO_CROSSWORD, 33, 1, 3, 33, 2, 1, 3)):
        assert lib.ss_acceptor_create(None, C.byref(bad), 16, C.byref(h)) == _lib.SS_ERR_INVALID_ARG and not h
    assert lib.ss_acceptor_create(None, C.byref(good), 0, C.byref(h)) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_create(None, None, 16, C.byref(h)) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_create(None, C.byref(good), 16, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_destroy(None) == _lib.SS_OK
    v = _lib.AcceptorView()
    assert lib.ss_acceptor_view_get(None, C.byref(v)) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_window_get(None, C.byref(h)) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_advance(None, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_accept(None, *([None, 0, None, None, None, 1, None, 0, None, None, 0] + [None] * 7)) == _lib.SS_ERR_INVALID_ARG


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_acceptor_create_without_device():
    lib = _lib.load()
    h = C.c_void_p()
    cfg = _lib.AcceptorConfig(_lib.SS_PROTO_CROSSWORD, 5, 0, 3, 5, 2, 1, 3)
    assert lib.ss_acceptor_create(None, C.byref(cfg), 16, C.byref(h)) == _lib.SS_ERR_NO_DEVICE and not h
    assert b"no CPU fallback" in lib.ss_last_error()


# ---------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------
def _t(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a).to(DEV)


def _buffer(rng, frames, odd=True):
    """frames back to back after random gaps, every frame at an odd offset"""
    offs, parts, at = [], [], 0
    for f in frames:
        gap = int(rng.integers(0, 24))
        if odd and (at + gap) % 2 == 0:
            gap += 1
        parts.append(bytes(rng.integers(0, 256, gap, dtype=np.uint8)))
        at += gap
        offs.append(at)
        parts.append(bytes(f))
        at += len(f)
    parts.append(bytes(rng.integers(0, 256, 16, dtype=np.uint8)))
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy(), np.array(offs, dtype=np.uint64)


def _acceptor(ctx, cfg, G):
    from summerset_b200.engine import Acceptor
    return Acceptor(ctx, cfg.protocol, G, cfg.n, cfg.me, cfg.d, cfg.T, cfg.av, cfg.wv, cfg.rv)


def _install(acc, st):
    acc.window_base.copy_(_t(np.array(st.base, dtype=np.uint64)))
    acc.bal_max_seen.copy_(_t(np.array(st.bmax, dtype=np.uint64)))


def _run_and_check(ctx, acc, cfg, st, frames, groups, peers, rng, store_cap=None, wal_cap=None, want_status=None):
    """one call on the device and in the model; compares verdicts, offsets, every byte of store / WAL / reply cells
    (canaries around every region and past the end) and the state words of every touched group"""
    buf, offs = _buffer(rng, frames)
    n = len(frames)
    big = 1 << 62
    # the model reads each frame where the kernel does: its length prefix decides where it ends inside the buffer
    mv = memoryview(buf.tobytes())
    frames_bytes = lambda i: bytes(mv[int(offs[i]):int(offs[i]) + want["dec"][i]["end"]])
    want = _stream(cfg, st, [mv[int(o):] for o in offs], groups, peers, big if store_cap is None else store_cap, big if wal_cap is None else wal_cap)
    s_tot, w_tot = want["totals"]
    s_size = (s_tot if store_cap is None else store_cap) + 64
    w_size = (w_tot if wal_cap is None else wal_cap) + 64
    s_can = rng.integers(0, 256, s_size, dtype=np.uint8)
    w_can = rng.integers(0, 256, w_size, dtype=np.uint8)
    store, wal = _t(s_can.copy()), _t(w_can.copy())
    out = acc.accept(_t(buf), _t(offs), _t(np.array(groups, dtype=np.uint32)), _t(np.array(peers, dtype=np.uint8)), store, wal,
                     s_tot if store_cap is None else store_cap, w_tot if wal_cap is None else wal_cap)
    status = ctx.device_status()
    if want_status is not None:
        assert status == want_status
    got = {k: v.cpu().numpy() for k, v in out.items()}
    assert [int(x) for x in got["verdict"].view(np.uint32)] == want["verdict"]
    assert [int(x) for x in got["store_off"].view(np.uint64)] == want["store_off"]
    assert [int(x) for x in got["wal_off"].view(np.uint64)] == want["wal_off"]
    assert [int(x) for x in got["wal_len"]] == want["wal_len"]
    assert [int(x) for x in got["totals"]] == list(want["totals"])
    assert [int(x) for x in got["reply_dst"]] == want["reply_dst"]
    # store and WAL: canary except the written bytes
    ws, ww = s_can.copy(), w_can.copy()
    for i in range(n):
        if want["verdict"][i] != ACC:
            continue
        f = want["dec"][i]
        at = want["store_off"][i]
        for s in f["shards"]:
            if s is None:
                continue
            ws[at:at + f["L"]] = np.frombuffer(s, dtype=np.uint8)
            ws[at + f["L"]:at + (f["L"] + 15) // 16 * 16] = 0
            at += _pitch(f["L"])
        rec = want["records"][i]
        ww[want["wal_off"][i]:want["wal_off"][i] + len(rec)] = np.frombuffer(rec, dtype=np.uint8)
        dec = pyoracle.decode_accept(rec, 1, cfg.cw)
        assert dec is not None and dec["slot"] == f["slot"] and dec["shards"] == f["shards"] and dec["variant"] == cfg.wv
    gs, gw = store.cpu().numpy(), wal.cpu().numpy()
    if not np.array_equal(gs, ws):
        bad = np.nonzero(gs != ws)[0]
        pytest.fail(f"store: {len(bad)} bytes differ, first at {bad[0]}")
    if not np.array_equal(gw, ww):
        bad = np.nonzero(gw != ww)[0]
        pytest.fail(f"wal: {len(bad)} bytes differ, first at {bad[0]}")
    # every record and reply against the oracle's independent encoders: a record re-encoded from the decoded fields
    # equals the device's wherever the frame itself is the canonical encoding of those fields (the record keeps the
    # frame's bytes verbatim, so a frame with non-minimal varints keeps them), and decodes back to those fields
    want["oracle_records"] = want["verbatim_only"] = 0
    for i in range(n):
        cell = got["replies"][i]
        if want["verdict"][i] != ACC:
            assert got["reply_len"][i] == 0 and not cell.any()
            continue
        f = want["dec"][i]
        rec = gw[want["wal_off"][i]:want["wal_off"][i] + int(got["wal_len"][i])].tobytes()
        dec = pyoracle.decode_accept(rec, 1, cfg.cw)
        assert dec is not None and dec["variant"] == cfg.wv, i
        assert (dec["slot"], dec["ballot"], dec["data_len"], dec["shard_len"], dec["shards"]) == \
            (f["slot"], f["ballot"], f["dlen"], f["L"], f["shards"]), i
        assert not cfg.cw or dec["assignment"] == f["asg"]
        if any(x is not None for x in f["shards"]):
            if frames_bytes(i) == _oracle_frame(pyoracle, cfg, f):
                assert rec == _oracle_record(pyoracle, cfg, f), i
                want["oracle_records"] += 1
            else:
                want["verbatim_only"] += 1
        r = _oracle_reply(pyoracle, cfg, f["slot"], st.inst[groups[i]][f["slot"]])
        assert r == want["replies"][i]
        assert got["reply_len"][i] == len(r) and cell[:len(r)].tobytes() == r, i
        assert not cell[len(r):].any()
    _check_state(acc, cfg, st, int(store.data_ptr()))
    return want, got


def _check_state(acc, cfg, st, store_ptr):
    torch.cuda.synchronize()
    G = len(st.base)
    assert [int(x) for x in acc.window_base.cpu().numpy().view(np.uint64)] == st.base
    assert [int(x) for x in acc.bal_max_seen.cpu().numpy().view(np.uint64)] == st.bmax
    accw = acc.accepting.cpu().numpy().view(np.uint64)
    ib = acc.inst_bal.cpu().numpy().view(np.uint64)
    src, held, dl = acc.source.cpu().numpy(), acc.held.cpu().numpy().view(np.uint32), acc.data_len.cpu().numpy().view(np.uint32)
    sa = acc.shard_addr.cpu().numpy().view(np.uint64)
    asg = acc.assignment.cpu().numpy().view(np.uint32) if cfg.cw else None
    for g in range(G):
        want_bits = 0
        for s, inst in st.inst[g].items():
            k = g * 64 + (s & 63)
            want_bits |= 1 << (s & 63)
            if "store_at" not in inst:
                continue
            assert (int(ib[k]), int(src[k]), int(held[k]), int(dl[k])) == (inst["bal"], inst["src"], inst["held"], inst["dlen"]), (g, s)
            if inst.get("fresh"):
                assert int(sa[k]) == store_ptr + inst["store_at"]
            if cfg.cw:
                assert int(asg[k]) == inst["asg"][cfg.me]
        assert int(accw[g]) == want_bits, g
    for g in range(G):
        for inst in st.inst[g].values():
            inst.pop("fresh", None)


# ---------------------------------------------------------------------------------------------
# GPU 1: frames from the real leader path
# ---------------------------------------------------------------------------------------------
LEADER_CASES = [("rspaxos", 5, 0, 0, True), ("crossword", 5, 5, 3, True), ("crossword", 5, 10, 6, True), ("crossword", 5, 5, 3, False),
                ("crossword", 5, 10, 6, False), ("rspaxos", 3, 0, 0, True), ("rspaxos", 12, 0, 0, True), ("crossword", 3, 6, 2, True),
                ("crossword", 7, 14, 7, False), ("crossword", 12, 24, 16, True), ("crossword", 12, 24, 16, False)]


def _leader_frames(ctx, oracle, rng, protocol, n, T, d, balanced, peer, lens=None, policies=None):
    """Accept frames for `peer` from the real leader path (LeaderEngine.propose_ragged -> frame_accept_pack_ragged), one
    per group, at random window bases and prepared ballots.  lens: the groups' request lengths (default: every varint
    edge plus a workload mix); policies: a Crossword policy table to use instead of the balanced / unbalanced ones."""
    from summerset_b200 import workloads as wl
    from summerset_b200.engine import LeaderEngine
    cw = protocol == "crossword"
    if lens is None:
        edges = [1, 2, 3, 250, 251, 750, 753, 65535, 65536, 196605, 196608, 4096, 1365, 1366]
        lens = np.concatenate([edges, wl.cfg4_lengths(150, seed_extra=7)[0]]).astype(np.uint32)
    lens = np.array(lens, dtype=np.uint32)
    rng.shuffle(lens)
    G = len(lens)
    eng = LeaderEngine(ctx, protocol, G, n, min(1, n - (n // 2 + 1)), 1, rs_total_shards=T, rs_data_shards=d)
    bal = rng.integers(1, 1 << 40, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    base = rng.integers(0, 1 << 40, G).astype(np.uint64)
    eng.window_base.copy_(_t(base))
    d, p, T = eng.d, eng.T - eng.d, eng.T
    if cw:
        if policies is not None:
            policies = np.array(policies, dtype=np.uint32)
        elif balanced:
            policies = np.stack([oracle.cw_brr_assignment(n, T, spr) for spr in range(T // n, d + 1, T // n)])
        else:
            full = (1 << T) - 1
            policies = np.array([[full & ~((1 << (T // n)) - 1) if r == 0 else (1 << (T // n)) - 1 if r == 1 else (1 << T) - 1 ^ (1 << r)
                                  for r in range(n)]], dtype=np.uint32)
        eng.set_policies([list(map(int, q)) for q in policies], balanced)
        pol = rng.integers(0, len(policies), G).astype(np.uint8)
    else:
        policies = np.array([[1 << r for r in range(n)]], dtype=np.uint32)
        pol = np.zeros(G, np.uint8)
    gaps = rng.integers(0, 32, G)
    ends = np.cumsum(lens.astype(np.int64) + gaps)
    data_off = (16 + ends - lens.astype(np.int64)).astype(np.uint64)
    arena = rng.integers(0, 256, 16 + int(ends[-1]) + 32, dtype=np.uint8)
    L = (lens.astype(np.int64) + d - 1) // d
    need = int(((L + 31) // 32 * 32).sum())
    store = torch.zeros((T, need + 32), dtype=torch.uint8, device=DEV)
    slot_out, shard_off, _ = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, _t(pol) if cw else None)
    out, off, fl, _ = ctx.frame_accept_pack_ragged(store, shard_off, _t(lens), d, p, policies, _t(pol), peer, slot_out, _t(bal),
                                                   with_assignment=cw)
    assert ctx.device_status() == 0
    out, off, fl = out.cpu().numpy(), off.cpu().numpy(), fl.cpu().numpy()
    frames = [out[int(off[g]):int(off[g]) + int(fl[g])].tobytes() for g in range(G)]
    eng.close()
    return frames, base, d, T


@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,T,d,balanced", LEADER_CASES)
def test_acceptor_takes_leader_frames(ctx, oracle, protocol, n, T, d, balanced):
    rng = np.random.default_rng(n * 100 + T + 7 * balanced)
    peer = 2
    frames, base, d, T = _leader_frames(ctx, oracle, rng, protocol, n, T, d, balanced, peer)
    G = len(frames)
    cfg = Cfg(protocol, n, peer, d, T)
    acc = _acceptor(ctx, cfg, G)
    st = State(G)
    st.base = [int(x) for x in base]
    _install(acc, st)
    groups = list(range(G))
    order = rng.permutation(G)
    want, _ = _run_and_check(ctx, acc, cfg, st, [frames[i] for i in order], [groups[i] for i in order], [0] * G, rng, want_status=0)
    assert want["verdict"].count(ACC) == sum(1 for f in frames if f) > G // 2
    assert want["verbatim_only"] == 0 and want["oracle_records"] == want["verdict"].count(ACC)
    acc.close()


# ---------------------------------------------------------------------------------------------
# GPU 2: adversarial batches against the model
# ---------------------------------------------------------------------------------------------
def _adversarial(oracle, rng, cfg, st, nfr):
    G = len(st.base)
    frames, groups, peers = [], [], []
    for _ in range(nfr):
        g = int(rng.integers(0, G + (1 if rng.random() < 0.02 else 0)))
        base = st.base[g] if g < G else 0
        r = rng.random()
        slot = base + int(rng.integers(0, 8))                 # repeated slots
        if r < 0.08:
            slot = max(base - 1 - int(rng.integers(0, 3)), 0)
        elif r < 0.14:
            slot = base + 64 + int(rng.integers(0, 4))
        bal = int(rng.integers(1, 12))
        dlen = int(rng.choice([1, 5, 40, 251, 700]))
        held = int(rng.integers(1, 1 << cfg.T))
        asg = [int(rng.integers(0, 1 << cfg.T)) for _ in range(cfg.n)] if cfg.cw else None
        f = _acc(oracle, slot, bal, held, dlen, cfg.d, cfg.T - cfg.d, asg, cfg.T, cfg.av)
        k = rng.random()
        if k < 0.04:
            f = f[:int(rng.integers(0, len(f)))]
        elif k < 0.07:
            f = oracle.frame_accept_reply(3, slot, bal, cfg.cw, 3)
        elif k < 0.08:
            f = b"\x00" * 7 + b"\x02" + b"\x01\x00"
        elif k < 0.10:
            f = _acc(oracle, slot, bal, held, dlen, cfg.d + 1, cfg.T - cfg.d - 1, asg, cfg.T, cfg.av)
        elif k < 0.20:                    # every varint in its 9-byte form: the shard offsets shift by 8 per shard
            f = _acc_wide(slot, bal, held, dlen, cfg.d, cfg.T - cfg.d, asg, cfg.T, cfg.av)
        frames.append(f)
        groups.append(g)
        peers.append(int(rng.integers(0, cfg.n)))
    return frames, groups, peers


@pytest.mark.gpu
@pytest.mark.parametrize("protocol", ["rspaxos", "crossword"])
def test_acceptor_adversarial_batches(ctx, oracle, protocol):
    cfg = Cfg(protocol, 5, 3, 3, 5) if protocol == "rspaxos" else Cfg(protocol, 5, 3, 3, 10)
    rng = np.random.default_rng(5 if protocol == "rspaxos" else 6)
    G = 37
    acc = _acceptor(ctx, cfg, G)
    st = State(G)
    st.base = [int(x) for x in rng.integers(0, 1 << 33, G)]
    st.bmax = [int(x) for x in rng.integers(0, 4, G)]
    _install(acc, st)
    counts = [0, 0]
    for rnd in range(4):
        frames, groups, peers = _adversarial(oracle, rng, cfg, st, 600)
        last = _acc(oracle, st.base[1], 1, 1, 700, cfg.d, cfg.T - cfg.d, [1] * cfg.n if cfg.cw else None, cfg.T)
        frames.append(last[:-40])         # runs past the end of the buffer
        groups.append(1)
        peers.append(0)
        if rnd == 0:                     # a stale-slot frame with the highest ballot first: it must not raise bal_max_seen
            frames.insert(0, _acc(oracle, st.base[0] - 1, 1 << 40, 1, 5, cfg.d, cfg.T - cfg.d,
                                  [1] * cfg.n if cfg.cw else None, cfg.T))
            groups.insert(0, 0)
            peers.insert(0, 1)
        want, _ = _run_and_check(ctx, acc, cfg, st, frames, groups, peers, rng, want_status=0)
        v = want["verdict"]
        for kind in (ACC, STALE_SLOT, STALE_BAL, BEYOND, MALFORMED, 3):
            assert kind in v, (rnd, hex(kind))
        counts[0] += want["oracle_records"]
        counts[1] += want["verbatim_only"]
        if rnd == 0:
            assert v[0] == STALE_SLOT and st.bmax[0] < 1 << 40
        upto = [b + int(rng.integers(0, 9)) for b in st.base]
        acc.advance(_t(np.array(upto, dtype=np.uint64)))
        _advance(st, upto)
    assert counts[0] > 100 and counts[1] >= 10, counts    # records re-encoded by the oracle / kept verbatim
    _check_state(acc, cfg, st, 0)
    acc.close()


# ---------------------------------------------------------------------------------------------
# GPU 3: store and WAL capacity
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which", ["store", "wal"])
def test_acceptor_capacity_cuts(ctx, oracle, which):
    cfg = Cfg("crossword", 5, 0, 3, 5)
    rng = np.random.default_rng(9)
    G = 60
    frames = [_acc(oracle, 0, 1, int(rng.integers(1, 32)), int(rng.integers(1, 3000)), 3, 2, CW_ROWS, 5) for _ in range(G)]
    full = _stream(cfg, State(G), frames, list(range(G)), [1] * G, 1 << 40, 1 << 40)
    k = 25
    if which == "store":
        edge = full["store_off"][k]                           # frames 0..k-1 fit exactly
        caps = [(edge, None), (edge - 1, None)]
    else:
        edge = full["wal_off"][k]
        caps = [(None, edge), (None, edge - 1)]
    for sc, wc in caps:
        acc = _acceptor(ctx, cfg, G)
        st = State(G)
        want, _ = _run_and_check(ctx, acc, cfg, st, frames, list(range(G)), [1] * G, rng, store_cap=sc, wal_cap=wc,
                                 want_status=STORE_FULL if which == "store" else FRAME_OVERFLOW)
        fit = k if (sc or wc) == edge else k - 1
        assert want["verdict"][:fit] == [ACC] * fit
        assert set(want["verdict"][fit:]) == {STORE_FULL_V if which == "store" else WAL_FULL_V}
        acc.close()


# ---------------------------------------------------------------------------------------------
# GPU 4: closed loop -- leader frames -> one acceptor per peer -> replies -> parse -> ingest -> tick, over windows
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,T", [pytest.param("rspaxos", 5, 0, id="rspaxos"), pytest.param("crossword", 5, 5, id="crossword")] +
                         [pytest.param("rspaxos", n, 0, id=f"rspaxos-{n}") for n in (3, 7, 9, 12)] +
                         [pytest.param("crossword", n, T, id=f"crossword-{n}-{T}") for n, T in ((3, 6), (7, 14), (12, 24))])
def test_acceptor_closed_loop(ctx, oracle, protocol, n, T):
    from summerset_b200 import workloads as wl
    from summerset_b200.engine import LeaderEngine
    f, G = 1, 300
    cw = protocol == "crossword"
    rng = np.random.default_rng((21 if cw else 22) + 100 * (n != 5) * (n + T))
    eng = LeaderEngine(ctx, protocol, G, n, f, 1, rs_total_shards=T, rs_data_shards=max(n // 2 + 1, T - 8) if cw else 0)
    bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    d, p, T = eng.d, eng.T - eng.d, eng.T
    if cw:
        policies = np.stack([oracle.cw_brr_assignment(n, T, spr) for spr in range(T // n, d + 1, T // n)])
        eng.set_policies([list(map(int, q)) for q in policies], True)
    else:
        policies = np.array([[1 << r for r in range(n)]], dtype=np.uint32)
    accs = {r: _acceptor(ctx, Cfg(protocol, n, r, d, T), G) for r in range(1, n)}
    majority = n // 2 + 1
    mb = np.zeros(G, dtype=np.int64)                    # model window base
    status = {}                                         # (g, slot) -> [acks set, committed]
    committed_total = 0
    for rnd in range(12):
        lens = np.where(rng.random(G) < 0.15, 0, wl.cfg4_lengths(G, seed_extra=rnd)[0] // 8 + 1).astype(np.uint32)
        pol = rng.integers(0, len(policies), G).astype(np.uint8) if cw else np.zeros(G, np.uint8)
        gaps = rng.integers(0, 32, G)
        ends = np.cumsum(lens.astype(np.int64) + gaps)
        data_off = (16 + ends - lens.astype(np.int64)).astype(np.uint64)
        arena = rng.integers(0, 256, 16 + int(ends[-1]) + 32, dtype=np.uint8)
        L = (lens.astype(np.int64) + d - 1) // d
        store = torch.zeros((T, int(((L + 31) // 32 * 32).sum()) + 32), dtype=torch.uint8, device=DEV)
        slot_out, shard_off, _ = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, _t(pol) if cw else None)
        ctx.device_status()
        slots = slot_out.cpu().numpy().view(np.uint64)
        for g in range(G):                               # first Null slot of the model's window
            first = next((s for s in range(int(mb[g]), int(mb[g]) + 64) if (g, s) not in status), None)
            want_slot = U64MAX if lens[g] == 0 or first is None else first
            assert int(slots[g]) == want_slot, (rnd, g)
        recs = []
        for g in range(G):                               # the leader's own AcceptData is durable: its self-ack
            if slots[g] != np.uint64(U64MAX):
                status[(g, int(slots[g]))] = [{0}, False, int(pol[g])]
                recs.append(oracle.frame_accept_reply(3, int(slots[g]), int(bal[g]), cw, 0))
        rec_group, rec_peer = [g for g in range(G) if slots[g] != np.uint64(U64MAX)], [0] * len(recs)
        for r, acc in accs.items():
            out, off, fl, _ = ctx.frame_accept_pack_ragged(store, shard_off, _t(lens), d, p, policies, _t(pol), r, slot_out, _t(bal),
                                                           with_assignment=cw)
            fl_h, off_h = fl.cpu().numpy(), off.cpu().numpy()
            sent = [g for g in range(G) if fl_h[g] > 0 and rng.random() < 0.8]      # some Accepts are lost
            buf_np = out.cpu().numpy()
            frames = [buf_np[int(off_h[g]):int(off_h[g]) + int(fl_h[g])].tobytes() for g in sent]
            buf, offs = _buffer(rng, frames)
            total = sum(((bin(int(policies[pol[g]][r])).count("1")) * _pitch(int(L[g]))) for g in sent) + 32
            astore = torch.empty(total, dtype=torch.uint8, device=DEV)
            awal = torch.empty(sum(len(x) + 32 for x in frames) + 32, dtype=torch.uint8, device=DEV)
            res = acc.accept(_t(buf), _t(offs), _t(np.array(sent, dtype=np.uint32)), _t(np.zeros(len(sent), np.uint8)), astore, awal)
            v = res["verdict"].cpu().numpy().view(np.uint32)
            assert (v == ACC).all(), rnd
            cells, rl, dst = res["replies"].cpu().numpy(), res["reply_len"].cpu().numpy(), res["reply_dst"].cpu().numpy()
            assert (dst == 0).all()
            for i, g in enumerate(sent):
                if rng.random() < 0.85:                  # some replies are lost too
                    recs.append(cells[i, :rl[i]].tobytes())
                    rec_group.append(g)
                    rec_peer.append(r)
        buf, offs = _buffer(rng, recs, odd=False)
        rg, rs_, rp, rb, rk = ctx.accept_reply_parse(_t(buf), _t(offs), _t(np.array(rec_group, dtype=np.uint32)),
                                                     _t(np.array(rec_peer, dtype=np.uint8)), eng.window_base, 3, cw)
        assert (rk.cpu().numpy() == 3).all()
        eng.on_accept_replies(rg, rs_, rp, rb)
        eng.tick()
        torch.cuda.synchronize()
        # the model: every reply names an Accepting instance of the leader's ballot
        for g, r, s in zip(rg.cpu().numpy(), rp.cpu().numpy(), rs_.cpu().numpy()):
            st_ = status[(int(g), int(mb[g]) + int(s))]
            st_[0].add(int(r))
        for (g, s), st_ in status.items():
            if st_[1] or s < mb[g]:
                continue
            acks = sum(1 << r for r in st_[0])
            if cw:
                ok = oracle.cw_committed(T, n, d, majority, f, acks, policies[st_[2]], True)
            else:
                ok = len(st_[0]) >= majority + f
            st_[1] = bool(ok)
        wbs = eng.window_base.cpu().numpy().view(np.uint64)
        cms = eng.committed.cpu().numpy().view(np.uint64)
        bars = eng.commit_bar.cpu().numpy()
        for g in range(G):
            prefix = 0
            while (g, int(mb[g]) + prefix) in status and status[(g, int(mb[g]) + prefix)][1] and prefix < 64:
                prefix += 1
            want_committed = sum(1 << i for i in range(64) if (g, int(mb[g]) + i) in status and status[(g, int(mb[g]) + i)][1])
            cm, r_ = int(cms[g]), int(wbs[g]) & 63
            cm_w = ((cm >> r_) | (cm << ((64 - r_) & 63))) & U64MAX
            assert cm_w == want_committed, (rnd, g)
            assert int(bars[g]) == prefix, (rnd, g)
        committed_total = sum(1 for x in status.values() if x[1])
        if rnd % 3 == 2:
            upto = mb + eng.commit_bar.cpu().numpy().astype(np.int64)
            eng.advance()
            for acc in accs.values():
                acc.advance(_t(upto.astype(np.uint64)))
            mb = upto
            torch.cuda.synchronize()
            assert (eng.window_base.cpu().numpy() == mb).all()
            for acc in accs.values():
                assert (acc.window_base.cpu().numpy() == mb).all()
    assert mb.max() >= 5 and committed_total > 0
    eng.close()
    for acc in accs.values():
        acc.close()
