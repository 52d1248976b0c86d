"""Reconstruct reads on the device acceptor (ss_acceptor_reconstruct_serve / ss_acceptor_absorb, summerset_b200/csrc/acceptor.cu).

`serve_model` restates handle_msg_reconstruct per message (rspaxos/messages.rs:468-516, crossword/messages.rs:577-632)
and `absorb_model` handle_msg_reconstruct_reply (rspaxos/messages.rs:519-594, crossword/messages.rs:635-722), over the
acceptor's state as `tests/test_acceptor_commit.Model` keeps it and its 64-slot window rule, with the stated differences
of the header comment.  Expected reply bytes are built from the oracle's encoders (varint, bitmap_encode and
ssor_rscodeword_encode); the GPU tests compare every reply byte, store byte and state word with the model, with
canaries around every output region, and run the closed loops leader -> acceptors -> commit -> reconstruct -> execute.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pyoracle
from summerset_b200 import _lib
from tests.test_acceptor import ACC, MALFORMED, STORE_FULL, STORE_FULL_V, FRAME_OVERFLOW, _buffer, _t, _vget
from tests.test_acceptor_commit import Model, Rig, _codeword, _pitch, _r16

NULL_V, RANGE_V, OUT_FULL_V = (_lib.SS_RECON_VERDICT_NULL_CODEWORD, _lib.SS_RECON_VERDICT_SHARD_RANGE,
                               _lib.SS_RECON_VERDICT_OUT_FULL)
RECON, REPLY = 4, 5
LENS = [1, 15, 16, 17, 250, 251, 65535, 65536]


def _bits(x):
    return [j for j in range(32) if (x >> j) & 1]


def _pc(x):
    return bin(x).count("1")


# ---------------------------------------------------------------------------------------------
# wire helpers: Reconstruct / ReconstructReply frames
# ---------------------------------------------------------------------------------------------
def _frame(body):
    return len(body).to_bytes(8, "big") + body


def _nm(v):
    """a non-minimal varint for v < 2^16 (tag 251 + u16), which the crate's decoder reads as v"""
    return bytes([251]) + v.to_bytes(2, "little")


def _var(v):
    """bincode's u64 varint, from the oracle's encoder"""
    return pyoracle.varint(v)


def bitmap_raw(size, blocks):
    """a Bitmap: the oracle's encoder for the layout it writes (one word per 64 bits, only the first non-zero), else by hand"""
    if size < 1 << 32 and len(blocks) == -(-size // 64) and not any(blocks[1:]):
        return pyoracle.bitmap_encode(size, blocks[0] if blocks else 0)
    return _var(size) + _var(len(blocks)) + b"".join(_var(b) for b in blocks)


def recon_frame(items, cw, variant=RECON):
    """items: RSPaxos slots, or Crossword (slot, size, blocks)"""
    body = _var(0) + _var(variant) + _var(len(items))
    for it in items:
        body += _var(it) if not cw else _var(it[0]) + bitmap_raw(it[1], it[2])
    return _frame(body)


def cw_bytes(d, p, dlen, L, shards, data_copy=None):
    """ssor_rscodeword_encode, with data_copy Some(bytes) appended by hand when given"""
    bufs = [None if s is None else np.frombuffer(bytes(s) + b"\0", dtype=np.uint8).copy() for s in shards]
    arr = (C.c_void_p * len(bufs))(*[None if b is None else b.ctypes.data for b in bufs])
    out = np.zeros(64 + len(shards) * (L + 16), dtype=np.uint8)
    lib = pyoracle.lib()
    lib.ssor_rscodeword_encode.restype = C.c_size_t
    n = lib.ssor_rscodeword_encode(d, p, C.c_uint64(dlen), C.c_uint64(L), arr, out.ctypes.data_as(C.c_void_p))
    b = out[:n].tobytes()
    assert b[-1] == 0
    return b if data_copy is None else b[:-1] + b"\x01" + bytes(data_copy)


def reply_frame(entries, d, T, variant=REPLY):
    """entries: (slot, bal, dlen, shards[T] bytes|None[, data_copy]) -> PeerMessage::Msg{ReconstructReply{slots_data}}"""
    body = _var(0) + _var(variant) + _var(len(entries))
    for e in entries:
        slot, bal, dlen, shards = e[:4]
        body += _var(slot) + _var(bal) + cw_bytes(d, T - d, dlen, -(-dlen // d), shards, e[4] if len(e) > 4 else None)
    return _frame(body)


def parse_reconstruct(frame, cw, variant=RECON):
    """-> list of items as recon_frame takes them, or the verdict of a frame that is not one"""
    if len(frame) < 8 or int.from_bytes(frame[:8], "big") != len(frame) - 8:
        return MALFORMED
    b = frame[8:]
    r = _vget(b, 0)
    if r is None:
        return MALFORMED
    if r[0] != 0:
        return 0x80000000 | r[0] if r[0] < 65536 else MALFORMED
    r = _vget(b, r[1])
    if r is None:
        return MALFORMED
    if r[0] != variant:
        return r[0] if r[0] < 65536 else MALFORMED
    r = _vget(b, r[1])
    if r is None:
        return MALFORMED
    cnt, n = r
    items = []
    for _ in range(cnt):
        r = _vget(b, n)
        if r is None:
            return MALFORMED
        slot, n = r
        if not cw:
            items.append(slot)
            continue
        vals = []
        for _ in range(2):
            r = _vget(b, n)
            if r is None:
                return MALFORMED
            vals.append(r[0])
            n = r[1]
        blocks = []
        for _ in range(vals[1]):
            r = _vget(b, n)
            if r is None:
                return MALFORMED
            blocks.append(r[0])
            n = r[1]
        items.append((slot, vals[0], blocks))
    return items if n == len(b) else MALFORMED


def flip_select(size, blocks, T):
    """Bitmap::decode + flip + subset_copy's walk and bound check -> (selected shards below T, an index >= T selected?).
    subset_copy iterates subset.iter(), which stops at Bitmap::size() = size as u8 (bitmap.rs:103-105, 258-270)."""
    walk = size % 256
    excl = lambda j: (blocks[j // 64] >> (j % 64)) & 1 if j // 64 < len(blocks) else 0
    bad = any(excl(j) == 0 for j in range(T, walk))
    sel = sum(1 << j for j in range(min(walk, T)) if not excl(j))
    return sel, bad


# ---------------------------------------------------------------------------------------------
# the per-message models
# ---------------------------------------------------------------------------------------------
def serve_model(m, cw, g, frame):
    """-> (verdict, reply bytes or None)"""
    items = parse_reconstruct(frame, cw) if g < m.G else MALFORMED
    if not isinstance(items, list):
        return items, None
    base, ent = m.base[g], {}
    for e, it in enumerate(items):
        slot = it if not cw else it[0]
        if slot < base or slot >= base + 64:
            continue
        inst = m.inst[g].get(slot)
        if inst is None:                                        # status < Accepting
            continue
        if cw:
            if inst["dlen"] == 0:
                return NULL_V, None
            sel, bad = flip_select(it[1], it[2], m.T)
            if bad:
                return RANGE_V, None
            mask = inst["held"] & sel
        else:
            mask = inst["held"]
        if mask:
            ent[slot] = (e, mask)
    if not ent:
        return ACC, None
    body = _var(0) + _var(REPLY) + _var(len(ent))
    for slot, (_, mask) in sorted(ent.items(), key=lambda kv: kv[1][0]):
        inst = m.inst[g][slot]
        L = -(-inst["dlen"] // m.d)
        sh = [inst["shards"][j] if (mask >> j) & 1 else None for j in range(m.T)]
        body += _var(slot) + _var(inst["bal"]) + cw_bytes(m.d, m.T - m.d, inst["dlen"], L, sh)
    return ACC, _frame(body)


def parse_reply(frame, d, T):
    """-> [(slot, bal, dlen, L, mask, shards)] or None when malformed under absorb's rules"""
    if len(frame) < 8 or int.from_bytes(frame[:8], "big") != len(frame) - 8:
        return None
    b = frame[8:]
    r = _vget(b, 0)
    if r is None or r[0] != 0:
        return r[0] if r is not None and r[0] < 65536 else None
    r = _vget(b, r[1])
    if r is None or r[0] != REPLY:
        return r[0] if r is not None and r[0] < 65536 else None
    cnt, n = _vget(b, r[1]) or (None, None)
    if cnt is None:
        return None
    out = []
    for _ in range(cnt):
        vals = []
        for _ in range(2):
            r = _vget(b, n)
            if r is None:
                return None
            vals.append(r[0])
            n = r[1]
        if len(b) - n < 2 or b[n] != d or b[n + 1] != T - d:
            return None
        n += 2
        for _ in range(3):
            r = _vget(b, n)
            if r is None:
                return None
            vals.append(r[0])
            n = r[1]
        slot, bal, dl, sl, t = vals
        if dl >= 1 << 32 or t != T or sl != -(-dl // d):
            return None
        mask, shards = 0, [None] * T
        for j in range(T):
            if n >= len(b) or b[n] > 1:
                return None
            n += 1
            if b[n - 1] == 0:
                continue
            r = _vget(b, n)
            if r is None or r[0] != sl or len(b) - r[1] < sl:
                return None
            n = r[1]
            shards[j] = bytes(b[n:n + sl])
            mask |= 1 << j
            n += sl
        if n >= len(b) or b[n] > 1:
            return None
        n += 1
        if b[n - 1] == 1:
            if len(b) - n < dl:
                return None
            n += dl
        out.append((slot, bal, dl, sl, mask, shards))
    return out if n == len(b) else None


def absorb_model(m, frames, groups, cap):
    """frames in call order -> (verdicts, absorbed counts, total, status); m takes the placed instances"""
    verdicts, counts, cur, contrib = [], [0] * len(frames), {}, []
    for fi, (fr, g) in enumerate(zip(frames, groups)):
        ents = parse_reply(fr, m.d, m.T) if g < m.G else None
        contrib.append([])
        if not isinstance(ents, list):
            verdicts.append(MALFORMED if ents is None else ents)
            continue
        verdicts.append(ACC)
        last = {e[0]: q for q, e in enumerate(ents)}            # a HashMap decode keeps the last insert
        base = m.base[g]
        for q, (slot, bal, dl, sl, mask, shards) in enumerate(ents):
            if last[slot] != q or slot < base or slot >= base + 64:
                continue
            inst = m.inst[g].get(slot)
            if inst is None or slot < m.eb[g] or bal < inst["bal"] or inst["dlen"] == 0 or dl != inst["dlen"]:
                continue
            have, sh = cur.get((g, slot), (inst["held"], list(inst["shards"])))
            add = mask & ~have
            if not add:
                continue
            for j in _bits(add):
                sh[j] = shards[j]
            cur[(g, slot)] = (have | add, sh)
            contrib[fi].append((g, slot))
    off, placed, status, regions = 0, set(), 0, []
    for g, slot in sorted(cur):
        mask, sh = cur[(g, slot)]
        sz = _pc(mask) * _pitch(-(-m.inst[g][slot]["dlen"] // m.d))
        if off + sz <= cap:
            placed.add((g, slot))
            m.inst[g][slot]["held"], m.inst[g][slot]["shards"] = mask, sh
            regions.append((g, slot, off))
        else:
            status |= STORE_FULL
        off += sz
    for fi, cs in enumerate(contrib):
        counts[fi] = sum(1 for k in cs if k in placed)
        if any(k not in placed for k in cs):
            verdicts[fi] = STORE_FULL_V
    return verdicts, counts, off, status, regions


# ---------------------------------------------------------------------------------------------
# CPU: the models on hand-written cases, symbols and refusals
# ---------------------------------------------------------------------------------------------
def _minst(m, g, s, bal, held, dlen, st="A"):
    shards = [bytes([j]) * (-(-dlen // m.d)) if (held >> j) & 1 else None for j in range(m.T)]
    m.inst[g][s] = dict(bal=bal, held=held, dlen=dlen, shards=shards, st=st)


def test_model_serve_rules(oracle):
    m = Model(1, 5, 1, 3, 5)
    m.base[0] = 100
    _minst(m, 0, 100, 7, 0b00010, 9)
    _minst(m, 0, 101, 7, 0b00110, 9, "C")
    _minst(m, 0, 102, 7, 0b00110, 0)                              # a null instance
    # RSPaxos: below the base, beyond the window and Null slots are skipped; a duplicate is one entry, ordered by its last
    v, r = serve_model(m, False, 0, recon_frame([99, 101, 164, 100, 150, 101], False))
    assert v == ACC
    want = _frame(_var(0) + _var(5) + _var(2) + _var(100) + _var(7) + cw_bytes(3, 2, 9, 3, [None, b"\1" * 3, None, None, None])
                  + _var(101) + _var(7) + cw_bytes(3, 2, 9, 3, [None, b"\1" * 3, b"\2" * 3, None, None]))
    assert r == want
    assert serve_model(m, False, 0, recon_frame([102], False))[0] == ACC and serve_model(m, False, 0, recon_frame([102], False))[1]
    assert serve_model(m, False, 0, recon_frame([99, 164], False)) == (ACC, None)
    # Crossword: held & flip(excl); an empty subset is skipped; the last non-empty occurrence defines the entry
    v, r = serve_model(m, True, 0, recon_frame([(101, 5, [0b00010]), (100, 5, [0]), (101, 5, [0b00110]), (101, 3, [0])], True))
    assert v == ACC and parse_reply(r, 3, 5) == [(100, 7, 9, 3, 0b00010, [None, b"\1" * 3, None, None, None]),
                                                 (101, 7, 9, 3, 0b00110, [None, b"\1" * 3, b"\2" * 3, None, None])]
    # narrower bitmap: bits beyond the size are not selected; wider: every bit of [T, size) must be set
    assert flip_select(2, [0], 5) == (0b11, False)
    assert flip_select(70, [~0 & (2**64 - 1) ^ 0b11111, 0b111111], 5) == (0b11111, False)
    assert flip_select(70, [(2**64 - 1) ^ 0b11111], 5)[1]                           # zero-padded block 1
    assert flip_select(6, [0], 5)[1] and not flip_select(6, [0b100000], 5)[1]
    assert flip_select(5, [0b11111, 0, 0], 5) == (0, False)                        # extra blocks are cut to the size
    # subset_copy walks [0, size mod 256): size 256 selects nothing, 256 + 5 walks the first five bits only
    assert flip_select(256, [0] * 4, 5) == (0, False) and flip_select(256, [], 5) == (0, False)
    assert flip_select(261, [0b00110], 5) == (0b11001, False) and flip_select(262, [0b11111], 5)[1]
    assert flip_select(262, [0b111111], 5) == (0, False)
    assert serve_model(m, True, 0, recon_frame([(100, 256, [0])], True)) == (ACC, None)
    assert serve_model(m, True, 0, recon_frame([(100, 300, [0])], True))[0] == RANGE_V
    assert serve_model(m, True, 0, recon_frame([(100, 6, [0])], True))[0] == RANGE_V
    assert serve_model(m, True, 0, recon_frame([(99, 6, [0]), (170, 6, [0])], True)) == (ACC, None)   # skipped first
    assert serve_model(m, True, 0, recon_frame([(102, 5, [0b11111])], True))[0] == NULL_V             # before the subset
    assert serve_model(m, True, 0, recon_frame([(103, 6, [0])], True)) == (ACC, None)                # Null: skipped
    assert serve_model(m, True, 0, _frame(b"\x00\x03\x00")) == (3, None)
    assert serve_model(m, True, 0, _frame(b"\x01")) == (0x80000001, None)
    assert serve_model(m, True, 0, recon_frame([(100, 5, [0])], True)[:-1]) == (MALFORMED, None)


def test_model_absorb_rules(oracle):
    m = Model(2, 5, 1, 3, 5)
    m.base = [10, 0]
    _minst(m, 0, 10, 5, 0b00010, 9, "C")
    _minst(m, 0, 11, 5, 0b00010, 9, "C")
    _minst(m, 0, 12, 5, 0b00010, 0, "C")                          # null: ignored
    _minst(m, 0, 13, 5, 0b00010, 9, "C")
    m.eb[0] = 11
    sh = lambda x: [bytes([x + j]) * 3 for j in range(5)]
    e = lambda s, bal, mask, x, dl=9: (s, bal, dl, [sh(x)[j] if (mask >> j) & 1 else None for j in range(5)])
    fr = [reply_frame([e(10, 5, 0b00101, 10), e(11, 9, 0b11111, 20), e(12, 5, 0b11111, 30), e(13, 4, 0b11111, 40),
                       e(9, 5, 0b1, 0), e(80, 5, 0b1, 0)], 3, 5),
          reply_frame([e(11, 5, 0b01100, 50), e(13, 5, 0b11111, 60, 10)], 3, 5),       # data_len mismatch
          reply_frame([e(11, 5, 0b00101, 70), e(11, 5, 0b01001, 80)], 3, 5),           # a repeated key: the last counts
          reply_frame([e(0, 1, 1, 0)], 3, 5)[:-1]]
    v, cnt, total, st, regions = absorb_model(m, fr, [0, 0, 0, 0], 1 << 20)
    assert v == [ACC, ACC, ACC, MALFORMED] and st == 0
    # slot 10 < exec_bar; 12 null; 13 stale ballot; 9 and 80 outside; slot 11 takes every shard from the first frame, so
    # the later frames add none; the held shard 1 stays as it was
    assert cnt == [1, 0, 0, 0] and m.inst[0][11]["held"] == 0b11111 and m.inst[0][11]["shards"][2] == sh(20)[2]
    assert m.inst[0][11]["shards"][1] == b"\1" * 3
    assert regions == [(0, 11, 0)] and total == 5 * 32
    _minst(m, 0, 14, 5, 0b00010, 9, "A")
    fr = [reply_frame([e(14, 5, 0b00101, 70), e(14, 5, 0b01001, 80)], 3, 5)]   # a repeated key: only the last counts
    v, cnt, total, st, regions = absorb_model(m, fr, [0], 1 << 20)
    assert cnt == [1] and m.inst[0][14]["held"] == 0b01011 and m.inst[0][14]["shards"][0] == sh(80)[0]
    # capacity: the second instance does not fit; a re-submission takes it
    _minst(m, 1, 0, 1, 0b1, 40, "C")
    _minst(m, 1, 1, 1, 0b1, 40, "C")
    fr = [reply_frame([(0, 1, 40, [None] + [bytes([7]) * 14] * 2 + [None] * 2), (1, 1, 40, [None] + [bytes([8]) * 14] * 2 + [None] * 2)], 3, 5)]
    v, cnt, total, st, _ = absorb_model(m, fr, [1], 3 * 32 + 16)
    assert v == [STORE_FULL_V] and cnt == [1] and st == STORE_FULL and total == 6 * 32 and m.inst[1][1]["held"] == 1
    v, cnt, total, st, _ = absorb_model(m, fr, [1], 3 * 32)
    assert v == [ACC] and cnt == [1] and total == 3 * 32 and m.inst[1][1]["held"] == 0b111


def test_reconstruct_symbols_and_refusals():
    lib = _lib.load()
    for name in ("ss_acceptor_reconstruct_serve", "ss_acceptor_absorb"):
        assert hasattr(lib, name)
    assert lib.ss_version() == 200
    assert lib.ss_acceptor_reconstruct_serve(None, None, 0, None, None, None, 1, 4, 5, None, 0, None, None, None, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_absorb(None, None, 0, None, None, None, 1, 5, None, 0, None, None, None) == _lib.SS_ERR_INVALID_ARG
    assert (NULL_V, RANGE_V, OUT_FULL_V) == (0xFFFFFFF6, 0xFFFFFFF7, 0xFFFFFFF8)


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_reconstruct_without_device():
    lib = _lib.load()
    h = C.c_void_p()
    cfg = _lib.AcceptorConfig(_lib.SS_PROTO_RSPAXOS, 5, 1, 3, 5, 2, 1, 3)
    assert lib.ss_acceptor_create(None, C.byref(cfg), 4, C.byref(h)) == _lib.SS_ERR_NO_DEVICE and not h


# ---------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------
class RRig(Rig):
    def serve(self, frames, groups, cap_delta=None):
        """serves frames; checks verdicts, offsets, every reply byte and the canaries against serve_model"""
        m = self.m
        want = [serve_model(m, self.cw, g, f) for f, g in zip(frames, groups)]
        sizes = [len(r) if r is not None and v == ACC else 0 for v, r in want]
        total = sum(_r16(s) for s in sizes)
        cap = total if cap_delta is None else total + cap_delta
        buf, offs = _buffer(self.rng, frames)
        canary = self.rng.integers(0, 256, max(cap, 0) + 64, dtype=np.uint8)
        out = _t(canary.copy())
        res = self.acc.reconstruct_serve(_t(buf), _t(offs), _t(np.array(groups, dtype=np.uint32)), _t(np.zeros(len(frames), np.uint8)),
                                         out, max(cap, 0))
        got = {k: v.cpu().numpy() for k, v in res.items()}
        exp = canary.copy()
        off, status = 0, 0
        ob = out.cpu().numpy()
        for i, ((v, r), s) in enumerate(zip(want, sizes)):
            gv, gl, go = int(got["verdict"][i]) & 0xFFFFFFFF, int(got["reply_len"][i]), int(got["reply_off"][i])
            if s and off + _r16(s) > cap:
                assert (gv, gl, go) == (OUT_FULL_V, 0, -1), i
                status |= FRAME_OVERFLOW
            elif s:
                assert (gv, gl, go) == (ACC, s, off), i
                assert ob[off:off + s].tobytes() == r, i
                exp[off:off + s] = np.frombuffer(r, dtype=np.uint8)
            else:
                assert (gv, gl, go) == (v, 0, -1), i
            off += _r16(s)
        assert int(got["total"][0]) == total
        if not np.array_equal(ob, exp):
            pytest.fail(f"serve output: {int((ob != exp).sum())} bytes differ")
        assert self.ctx.device_status() == status
        self.check_state()
        return want, got

    def absorb(self, frames, groups, cap=None, store=None, pad=0):
        """pad: that many other-message frames (PeerMsg variant 3) ahead of frames, which must come back untouched"""
        m = self.m
        snap = Model(m.G, m.n, m.me, m.d, m.T)
        snap.base, snap.eb = list(m.base), list(m.eb)
        snap.inst = [{s: dict(v, shards=list(v["shards"])) for s, v in d.items()} for d in m.inst]
        need = absorb_model(snap, frames, groups, 1 << 62)[2]
        cap = need if cap is None else cap
        verdicts, counts, total, status, regions = absorb_model(m, frames, groups, cap)
        assert total == need
        canary = self.rng.integers(0, 256, cap + 64, dtype=np.uint8)
        st = _t(canary.copy()) if store is None else store
        self.stores.append(st)
        buf, offs = _buffer(self.rng, frames)
        grp = np.array(groups, dtype=np.uint32)
        if pad:
            pf = np.frombuffer(_frame(b"\x00\x03"), dtype=np.uint8)
            offs = np.concatenate([np.arange(pad, dtype=np.uint64) * np.uint64(len(pf)), offs + np.uint64(pad * len(pf))])
            buf = np.concatenate([np.tile(pf, pad), buf])
            grp = np.concatenate([np.zeros(pad, np.uint32), grp])
        res = self.acc.absorb(_t(buf), _t(offs), _t(grp), _t(np.zeros(len(grp), np.uint8)), st, cap)
        got = {k: v.cpu().numpy() for k, v in res.items()}
        assert (got["verdict"][:pad] == 3).all() and (got["absorbed"][:pad] == 0).all()
        got["verdict"], got["absorbed"] = got["verdict"][pad:], got["absorbed"][pad:]
        assert [int(x) & 0xFFFFFFFF for x in got["verdict"]] == verdicts
        assert [int(x) for x in got["absorbed"]] == counts
        assert int(got["total"][0]) == total
        assert self.ctx.device_status() == status
        exp = canary.copy()
        for g, s, off in regions:
            inst = m.inst[g][s]
            L = -(-inst["dlen"] // m.d)
            for k, j in enumerate(_bits(inst["held"])):
                exp[off + k * _pitch(L):off + k * _pitch(L) + _r16(L)] = 0
                exp[off + k * _pitch(L):off + k * _pitch(L) + L] = np.frombuffer(inst["shards"][j], dtype=np.uint8)
        ob = st.cpu().numpy()
        if not np.array_equal(ob, exp):
            pytest.fail(f"absorb store: {int((ob != exp).sum())} bytes differ")
        held = self.acc.held.cpu().numpy().view(np.uint32)
        addr = self.acc.shard_addr.cpu().numpy().view(np.uint64)
        for g in range(m.G):
            for s, inst in m.inst[g].items():
                assert int(held[g * 64 + (s & 63)]) == inst["held"], (g, s)
        for g, s, off in regions:
            assert int(addr[g * 64 + (s & 63)]) == st.data_ptr() + off
        self.check_state()
        return verdicts, counts


def _fill(rig, items_per_group, rng, d, T, base=None, held_fn=None, lens=LENS):
    """accepts instances at window slots, commits every other one; returns the slots per group"""
    G = rig.m.G
    if base is not None:
        rig.set_base(base)
    items = []
    for g in range(G):
        for k in range(items_per_group):
            s = rig.m.base[g] + k * 3 % 64
            if any(it[0] == g and it[1] == s for it in items):
                continue
            dlen = int(lens[(g + k) % len(lens)])
            dlen = max(1, dlen * d // 4) if dlen > 4096 and d > 4 else dlen
            data, sh = _codeword(rng, dlen, d, T)
            h = held_fn(g, k) if held_fn else int(rng.integers(1, 1 << T))
            items.append((g, s, int(rng.choice([1, 200, 300, 70000, 1 << 33])), h, data, sh))
    rig.accept(items)
    return items


def _serve_frames(rig, rng, cw, T, nfr):
    frames, groups = [], []
    for _ in range(nfr):
        g = int(rng.integers(0, rig.m.G))
        base = rig.m.base[g]
        items = []
        for _ in range(int(rng.integers(0, 6))):
            s = base + int(rng.integers(-3, 70)) if base >= 3 else base + int(rng.integers(0, 70))
            if not cw:
                items.append(s)
                continue
            kind = int(rng.integers(0, 10))
            if kind < 6:
                items.append((s, T, [int(rng.integers(0, 1 << T))]))
            elif kind < 8:
                items.append((s, int(rng.integers(1, T + 1)), [int(rng.integers(0, 1 << 63))]))     # narrower
            elif kind == 8:
                sz = T + int(rng.integers(1, 100))                                                    # wider, all set
                items.append((s, sz, [((1 << 64) - 1) & ~((1 << T) - 1) | int(rng.integers(0, 1 << T))] + [(1 << 64) - 1] * ((sz - 1) // 64)))
            else:                                  # wider: refused unless every walked bit >= T is set; walks stop at size mod 256
                sz = int(rng.choice([T + 1, 256, 256 + T, 257 + T, 600]))
                blk = int(rng.integers(0, 1 << T)) | (int(rng.integers(0, 2)) << T)
                items.append((s, sz, [blk] + [0] * int(rng.integers(0, 3))))
        if items and rng.integers(0, 3) == 0:
            items.append(items[0])                                                                    # a duplicate
        frames.append(recon_frame(items, cw))
        groups.append(g)
    return frames, groups


# ---------------------------------------------------------------------------------------------
# GPU: serve
# ---------------------------------------------------------------------------------------------
SERVE_CODES = ([("rspaxos", n, n // 2 + 1, n) for n in range(1, 33)] + [("crossword", n, max(1, n // 2), n) for n in range(1, 33)]
               + [("crossword", 32, d, 32) for d in (1, 16, 31, 32)])


@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,d,T", [(p, n, d, T) for p, n, d, T in SERVE_CODES])
def test_serve(ctx, protocol, n, d, T):
    cw = protocol == "crossword"
    rig = RRig(ctx, protocol, 6, n, n - 1, d, T)
    rng = rig.rng
    _fill(rig, 5, rng, d, T, base=[0, 3, 250, 65535, 1 << 20, (1 << 33) + 5])
    rig.commit_all()
    rig.execute(check_data=False)
    frames, groups = _serve_frames(rig, rng, cw, T, 40)
    frames += [_frame(b"\x00\x02\x00"), _frame(b"\x02"), _frame(recon_frame([0] if not cw else [(0, 5, [0])], cw)[8:-1]),
               _frame(_var(0) + _var(4) + _var(1) + _nm(rig.m.base[1]) + (bitmap_raw(T, [0]) if cw else b""))]
    groups += [0, 1, 2, 1]
    frames.append(recon_frame([1], cw) if not cw else recon_frame([(1, T, [0])], cw))
    groups.append(7)                                                                                  # group >= G
    rig.serve(frames, groups)


@pytest.mark.gpu
@pytest.mark.parametrize("protocol", ["rspaxos", "crossword"])
def test_serve_null_capacity_and_lengths(ctx, protocol):
    cw = protocol == "crossword"
    n, d, T = 5, 3, 5
    rig = RRig(ctx, protocol, len(LENS) + 1, n, 1, d, T)
    rng = rig.rng
    items = []
    for g, L in enumerate(LENS):
        data, sh = _codeword(rng, L * d, d, T)
        items.append((g, 0, 9, 0b10110, data, sh))
    items.append((len(LENS), 0, 9, 0b00010, b"", [b""] * T))                    # a null instance: RSPaxos serves it
    rig.accept(items)
    frames = [recon_frame([0], cw) if not cw else recon_frame([(0, T, [0b00100])], cw) for _ in range(len(LENS) + 1)]
    groups = list(range(len(LENS) + 1))
    want, _ = rig.serve(frames, groups)
    assert want[-1][0] == (NULL_V if cw else ACC)
    tot = sum(_r16(len(r)) for v, r in want if r)
    for delta in (0, -1):                                                      # exact, then one byte short
        rig.serve(frames, groups, cap_delta=delta)
    assert tot > 0


# ---------------------------------------------------------------------------------------------
# GPU: absorb
# ---------------------------------------------------------------------------------------------
def _reply_entries(rig, rng, g, all_shards, nent, stale=False):
    m = rig.m
    base = m.base[g]
    ents = []
    for _ in range(nent):
        s = base + int(rng.integers(-2 if base >= 2 else 0, 68))
        inst = m.inst[g].get(s)
        dlen, sh = all_shards.get((g, s), (int(rng.integers(1, 40)), None))
        if sh is None:
            _, sh = _codeword(rng, dlen, m.d, m.T)
        kind = int(rng.integers(0, 10))
        if kind == 0 and inst is not None:                                     # data_len mismatch
            dlen2 = dlen + m.d
            _, sh = _codeword(rng, dlen2, m.d, m.T)
            dlen = dlen2
        elif kind == 1:                                                        # different bytes for the same shards
            sh = [bytes(rng.integers(0, 256, len(x), dtype=np.uint8)) for x in sh]
        bal = (inst["bal"] if inst else 1) + int(rng.integers(-1 if stale else 0, 2))
        mask = int(rng.integers(0, 1 << m.T))
        e = (s, max(bal, 0), dlen, [sh[j] if (mask >> j) & 1 else None for j in range(m.T)])
        if rng.integers(0, 4) == 0:
            e = e + (bytes(rng.integers(0, 256, dlen, dtype=np.uint8)),)     # data_copy: Some(data_len bytes)
        ents.append(e)
    return ents


def _raw_entry_frame(slot, bal, dd, pp, dlen, sl, count, shard_len=None):
    """one entry with every codeword field as given: count present shards of shard_len (default sl) bytes"""
    sb = sl if shard_len is None else shard_len
    body = _var(0) + _var(REPLY) + _var(1) + _var(slot) + _var(bal) + bytes([dd, pp]) + _var(dlen) + _var(sl) + _var(count)
    body += b"".join(b"\x01" + _var(sb) + bytes([j]) * sb for j in range(count)) + b"\x00"
    return _frame(body)


def _codeword_rule_frames(m, shards, g, d, T):
    """a frame that breaks exactly one codeword rule, each aimed at a live instance: all malformed"""
    s = sorted(m.inst[g])[0]
    dlen = shards[(g, s)][0]
    L, bal = -(-dlen // d), m.inst[g][s]["bal"]
    ok = _raw_entry_frame(s, bal, d, T - d, dlen, L, T)
    assert parse_reply(ok, d, T) is not None                                  # the unbroken frame decodes
    return [_raw_entry_frame(s, bal, d + 1 if d < T else d - 1, T - d, dlen, L, T),    # d alone
            _raw_entry_frame(s, bal, d, T - d + 1, dlen, L, T),                         # p alone
            _raw_entry_frame(s, bal, d, T - d, dlen, L + 1, T),                         # shard_len != ceil(data_len / d)
            _raw_entry_frame(s, bal, d, T - d, dlen, L, T + 1),                         # T + 1 shard Options
            _raw_entry_frame(s, bal, d, T - d, dlen, L, T, L + 1)]                      # a shard of another length


def _nm_reply(m, shards, g, d, T):
    """one entry carrying every shard of group g's first instance, every small varint non-minimal"""
    nmv = lambda v: _nm(v) if v < 65536 else _var(v)
    s = sorted(m.inst[g])[0]
    dlen, sh = shards[(g, s)]
    L = -(-dlen // d)
    body = _nm(0) + _nm(REPLY) + _nm(1) + nmv(s) + nmv(m.inst[g][s]["bal"]) + bytes([d, T - d]) + nmv(dlen) + nmv(L) + _nm(T)
    body += b"".join(b"\x01" + nmv(L) + sh[j] for j in range(T)) + b"\x00"
    return _frame(body)


@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,d,T", [("rspaxos", 5, 3, 5), ("crossword", 5, 3, 5), ("crossword", 7, 7, 14), ("crossword", 3, 1, 3),
                                            ("crossword", 32, 16, 32), ("crossword", 32, 31, 32)])
def test_absorb(ctx, protocol, n, d, T):
    rig = RRig(ctx, protocol, 9, n, 1, d, T)
    rng = rig.rng
    items = _fill(rig, 6, rng, d, T, base=[0, 5, 300, 70000, 1 << 34, 0, 2, 64, 0], lens=[1, 15, 17, 251, 600, 3000])
    shards = {(g, s): (len(data), sh) for g, s, _, _, data, sh in items}
    rig.commit_all()
    rig.m.eb[3] = rig.m.base[3] + 3
    rig.acc.exec_bar.copy_(_t(np.array(rig.m.eb, dtype=np.uint64)))
    for rnd in range(3):                                                        # scratch regrown across calls
        frames, groups = [], []
        for _ in range(4 + 30 * rnd):
            g = int(rng.integers(0, 9)) if rnd < 2 else 4                     # the last round: many frames for one group
            ents = _reply_entries(rig, rng, g, shards, int(rng.integers(0, 5)), stale=True)
            if ents and rng.integers(0, 4) == 0:
                ents.append(ents[0][:1] + ents[-1][1:])                        # a repeated key
            frames.append(reply_frame(ents, d, T))
            groups.append(g)
        frames += [_frame(b"\x00\x03"), _frame(reply_frame(_reply_entries(rig, rng, 1, shards, 1), d, T)[8:-1]),
                   reply_frame(_reply_entries(rig, rng, 0, shards, 2), d, T - 1), _nm_reply(rig.m, shards, 0, d, T)]
        frames += _codeword_rule_frames(rig.m, shards, 0, d, T)
        groups += [0] * (len(frames) - len(groups))
        rig.absorb(frames, groups)
    rig.execute(check_data=False)


@pytest.mark.gpu
def test_absorb_first_wins_capacity_and_drain(ctx):
    n, d, T = 5, 3, 5
    rig = RRig(ctx, "crossword", 40, n, 2, d, T)
    rng = rig.rng
    items = []
    for g in range(40):
        for s in range(2):
            data, sh = _codeword(rng, int(rng.integers(1, 3000)), d, T)
            items.append((g, s, 3, 0b00100, data, sh))
    rig.accept(items)
    rig.commit_all()
    sh_of = {(it[0], it[1]): it[5] for it in items}
    dl_of = {(it[0], it[1]): len(it[4]) for it in items}
    frames, groups = [], []
    for g in range(40):
        for peer, mask in ((0, 0b00011), (1, 0b00110)):                      # shard 1 from two frames, different bytes
            ents = []
            for s in range(2):
                sh = [x if peer == 0 else bytes(255 - b for b in x) for x in sh_of[(g, s)]]
                ents.append((s, 3, dl_of[(g, s)], [sh[j] if (mask >> j) & 1 else None for j in range(T)]))
            frames.append(reply_frame(ents, d, T))
            groups.append(g)
    need = sum(3 * _pitch(-(-dl_of[k] // d)) for k in sh_of)
    edge = sum(3 * _pitch(-(-dl_of[(g, s)] // d)) for g in range(13) for s in range(2))
    v, _ = rig.absorb(frames, groups, cap=edge - 1)
    assert v.count(STORE_FULL_V) > 0 and rig.m.inst[12][1]["held"] == 0b00100
    calls = 0
    while any(rig.m.inst[g][s]["held"] != 0b00111 for g in range(40) for s in range(2)):
        rig.absorb(frames, groups, cap=edge)
        calls += 1
    assert calls >= 2 and need > edge
    for g in range(40):                                                        # the first frame's shard 1 won
        assert rig.m.inst[g][0]["shards"][1] == sh_of[(g, 0)][1]
    recs, st = rig.execute()
    assert len(recs) == 80 and st == 0


@pytest.mark.gpu
def test_absorb_exec_bar_and_stale_ballot(ctx):
    """slots below exec_bar count as Executed and an entry below inst.bal is stale: neither absorbs anything"""
    n, d, T = 5, 3, 5
    rig = RRig(ctx, "crossword", 2, n, 2, d, T)
    rng = rig.rng
    items = []
    for g in range(2):
        for s in range(4):
            data, sh = _codeword(rng, 100 + 7 * s, d, T)
            items.append((g, s, 3, 0b00100, data, sh))
    rig.accept(items)
    rig.commit_all()
    rig.m.eb = [2, 0]
    rig.acc.exec_bar.copy_(_t(np.array(rig.m.eb, dtype=np.uint64)))
    frames = [reply_frame([(s, 2 if s == 3 else 3, len(items[4 * g + s][4]), [x if j != 2 else None for j, x in enumerate(items[4 * g + s][5])])
                           for s in range(4)], d, T) for g in range(2)]
    _, cnt = rig.absorb(frames, [0, 1])
    assert cnt == [1, 3]
    assert [rig.m.inst[0][s]["held"] for s in range(4)] == [0b00100, 0b00100, 0b11111, 0b00100]


def _warp_cap(ctx):
    return ctx.sm_count * 64 * 8          # launch_grid: 64 CTAs per SM, 8 warps per CTA: frames / segments per sweep


def _thread_cap(ctx):
    return ctx.sm_count * 64 * 256        # absorb_decode_kernel: a thread per frame


@pytest.mark.gpu
@pytest.mark.parametrize("protocol", ["rspaxos", "crossword"])
def test_serve_past_the_grid_cap(ctx, protocol):
    """more frames than serve_count / serve_copy have warps: later frames take a warp's second sweep and reuse its
    shared tables, each reply checked byte for byte"""
    cw = protocol == "crossword"
    n, d, T = 3, 2, 3
    rig = RRig(ctx, protocol, 64, n, 1, d, T)
    rng = rig.rng
    _fill(rig, 4, rng, d, T, base=[int(x) for x in rng.integers(0, 1 << 20, 64)], lens=[1, 5, 17, 40])
    rig.commit_all()
    N = _warp_cap(ctx) + 1000
    frames, groups = [], []
    for i in range(N):
        g = i % 64
        base = rig.m.base[g]
        slots = [base + int(x) * 3 for x in rng.integers(0, 5, 1 + i % 3)]
        frames.append(recon_frame([(s, T, [int(rng.integers(0, 1 << T))]) for s in slots] if cw else slots, cw))
        groups.append(g)
    want, got = rig.serve(frames, groups)
    assert sum(1 for v, r in want[-1000:] if r) > 200                      # replies in the second sweep


@pytest.mark.gpu
def test_absorb_past_the_grid_caps(ctx):
    """one reply frame for each of more groups than absorb_plan / absorb_copy have warps, so segment heads come past the
    first sweep, behind more other-message frames than absorb_decode has threads"""
    n, d, T, me = 5, 3, 5, 1
    G = _warp_cap(ctx) + 1000
    rig = RRig(ctx, "rspaxos", G, n, me, d, T)
    rng = rig.rng
    live = [g for g in range(G) if g % 97 == 0 or g >= G - 600]
    shards, items = {}, []
    for g in live:
        data, sh = _codeword(rng, 1 + g % 50, d, T)
        shards[g] = (len(data), sh)
        items.append((g, 0, 2, 1 << me, data, sh))
    rig.accept(items)
    rig.commit_all()
    idle = reply_frame([(0, 2, 10, [b"\x07" * 4] * T)], d, T)                 # slot 0 of a group with no instance: ignored
    frames = [reply_frame([(0, 2, shards[g][0], [x if j != me else None for j, x in enumerate(shards[g][1])])], d, T) if g in shards
              else idle for g in range(G)]
    _, cnt = rig.absorb(frames, list(range(G)), pad=_thread_cap(ctx) + 1000)
    assert sum(cnt) == len(live)
    recs, st = rig.execute()
    assert len(recs) == len(live) and st == 0


@pytest.mark.gpu
def test_reconstruct_null_pointers(ctx):
    rig = RRig(ctx, "rspaxos", 2, 5, 1, 3, 5)
    lib, h = rig.acc.lib, rig.acc.h
    x = torch.zeros(64, dtype=torch.uint8, device="cuda")
    p = x.data_ptr()
    assert lib.ss_acceptor_reconstruct_serve(h, p, 64, p, p, None, 1, 4, 5, p, 64, p, p, p, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_reconstruct_serve(h, p, 64, p, p, p, 1, 4, 5, p + 1, 64, p, p, p, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_absorb(h, p, 64, p, p, p, 1, 5, None, 64, p, p, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_absorb(h, p, 64, p, p, p, 1, 5, p + 8, 64, p, p, None) == _lib.SS_ERR_INVALID_ARG
    assert lib.ss_acceptor_absorb(h, None, 0, None, None, None, 0, 5, None, 0, None, None, None) == _lib.SS_OK


# ---------------------------------------------------------------------------------------------
# GPU: closed loops through the leader path
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("protocol,n,T,d,spr", [("crossword", 5, 5, 3, 1), ("crossword", 5, 5, 3, 2), ("crossword", 7, 14, 7, 2),
                                                 ("rspaxos", 5, 5, 3, 1)])
def test_closed_loop_reconstruct(ctx, oracle, protocol, n, T, d, spr):
    from summerset_b200 import workloads as wl
    from summerset_b200.engine import Acceptor, LeaderEngine
    cw = protocol == "crossword"
    G = 64
    rng = np.random.default_rng(n * 100 + T + spr)
    eng = LeaderEngine(ctx, protocol, G, n, 1, 1, **(dict(rs_total_shards=T, rs_data_shards=d) if cw else {}))
    d, p, T = eng.d, eng.T - eng.d, eng.T
    bal = rng.integers(1, 1 << 30, G).astype(np.uint64)
    eng.set_prepared_ballots(_t(bal))
    if cw:
        policies = np.array([oracle.cw_brr_assignment(n, T, spr)], dtype=np.uint32)
        eng.set_policies([list(map(int, q)) for q in policies], False)
    else:
        policies = np.array([[1 << r for r in range(n)]], dtype=np.uint32)
    accs = [Acceptor(ctx, protocol, G, n, r, d, T) for r in range(n)]
    keep, delivered = [], 0
    me = 1
    for rnd in range(3):
        lens = (wl.cfg4_lengths(G, seed_extra=rnd)[0] // 4 + rng.integers(0, 7, G)).astype(np.uint32)
        gaps = rng.integers(0, 32, G)
        ends = np.cumsum(lens.astype(np.int64) + gaps)
        data_off = (16 + ends - lens.astype(np.int64)).astype(np.uint64)
        arena = rng.integers(0, 256, 16 + int(ends[-1]) + 32, dtype=np.uint8)
        L = (lens.astype(np.int64) + d - 1) // d
        store = torch.zeros((T, int(((L + 31) // 32 * 32).sum()) + 32), dtype=torch.uint8, device="cuda")
        pol = np.zeros(G, np.uint8)
        slot_out, shard_off, _ = eng.propose_ragged(_t(arena), _t(data_off), _t(lens), store, _t(pol) if cw else None)
        slots = slot_out.cpu().numpy().view(np.uint64)
        for r, acc in enumerate(accs):
            out, off, fl, _ = ctx.frame_accept_pack_ragged(store, shard_off, _t(lens), d, p, policies, _t(pol), r, slot_out, _t(bal),
                                                           with_assignment=cw)
            off_h, fl_h, ob = off.cpu().numpy(), fl.cpu().numpy(), out.cpu().numpy()
            frames = [ob[int(off_h[g]):int(off_h[g]) + int(fl_h[g])].tobytes() for g in range(G)]
            buf, offs = _buffer(rng, frames)
            astore = torch.empty(sum(len(f) for f in frames) * 2 + 64, dtype=torch.uint8, device="cuda")
            awal = torch.empty(sum(len(f) + 48 for f in frames) + 64, dtype=torch.uint8, device="cuda")
            keep.append(astore)
            res = acc.accept(_t(buf), _t(offs), _t(np.arange(G, dtype=np.uint32)), _t(np.zeros(G, np.uint8)), astore, awal)
            assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
            acc.heartbeat(_t(np.arange(G, dtype=np.uint32)), _t(np.zeros(G, np.uint8)), _t(bal), _t(slots + np.uint64(1)),
                          _t(np.zeros(G, np.uint64)))
        sent = [arena[int(data_off[g]):int(data_off[g]) + int(lens[g])].tobytes() for g in range(G)]
        fol = accs[me]
        held_me = int(policies[0][me])
        outb = torch.empty(int(sum(_r16(int(x)) for x in lens)) + 16, dtype=torch.uint8, device="cuda")
        ex = fol.execute(outb, G)
        assert int(ex["totals"][0].item()) == (G if _pc(held_me) >= d else 0)
        if _pc(held_me) >= d:
            continue
        # the requests: Crossword gossip targets and exclusions; RSPaxos step-up asks every peer
        reqs = {}
        for g in range(G):
            if cw:
                t, excl = oracle.gossip_targets_excl(me, n, d, 0, held_me, policies[0], (1 << n) - 1)
                for q in _bits(t):
                    reqs.setdefault(q, []).append((g, recon_frame([(int(slots[g]), T, [int(excl[q])])], True)))
            else:
                for q in range(n):
                    if q != me:
                        reqs.setdefault(q, []).append((g, recon_frame([int(slots[g])], False)))
        replies, rgroups = [], []
        for q, lst in sorted(reqs.items()):
            buf, offs = _buffer(rng, [f for _, f in lst])
            out = torch.empty(1 << 22, dtype=torch.uint8, device="cuda")
            res = accs[q].reconstruct_serve(_t(buf), _t(offs), _t(np.array([g for g, _ in lst], dtype=np.uint32)),
                                            _t(np.full(len(lst), me, np.uint8)), out)
            assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all()
            ro, rl, ob = res["reply_off"].cpu().numpy(), res["reply_len"].cpu().numpy(), out.cpu().numpy()
            for k, (g, _) in enumerate(lst):
                assert rl[k] > 0
                replies.append(ob[int(ro[k]):int(ro[k]) + int(rl[k])].tobytes())
                rgroups.append(g)
        buf, offs = _buffer(rng, replies)
        fstore = torch.empty(1 << 24, dtype=torch.uint8, device="cuda")
        keep.append(fstore)
        res = fol.absorb(_t(buf), _t(offs), _t(np.array(rgroups, dtype=np.uint32)), _t(np.zeros(len(replies), np.uint8)), fstore)
        assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all() and ctx.device_status() == 0
        assert (np.bincount(rgroups, weights=res["absorbed"].cpu().numpy(), minlength=G) >= 1).all()
        ex = fol.execute(outb, G)
        assert ctx.device_status() == 0 and int(ex["totals"][0].item()) == G
        ob = outb.cpu().numpy()
        for k in range(G):
            g, s, o, ln = int(ex["rec_group"][k]), int(ex["rec_slot"][k]), int(ex["rec_off"][k]), int(ex["rec_len"][k])
            assert (g, s) == (k, int(slots[k])) and ob[o:o + ln].tobytes() == sent[g]
            delivered += 1
        upto = _t(slots.astype(np.uint64) + np.uint64(1))
        for acc in accs:
            acc.advance(upto)
        eng.advance(None)
    assert delivered == (3 * G if _pc(int(policies[0][me])) < d else 0)
    eng.close()
    for acc in accs:
        acc.close()
