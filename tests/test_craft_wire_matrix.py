"""Every CRaft frame and record the device reads or writes, at every variant index and varint width the ABI accepts.

The CRaft calls take their bincode enum indices (PeerMsg and DurEntry variants) as arguments.  A varint below 251 is one
byte, below 2^16 three bytes, so every offset after a variant shifts with its width; terms, slots and conflict fields
shift the same way at 251, 2^16 and 2^32.  The tests below run the follower's append, the leader's pack / reply parse /
back-off loop, the elections, step-down and the reconstruct reads at settings that cover each width, each setting one
tuple for every variant of the path, and put follower rings and terms across each field width edge.  The restatements
are those of tests/test_follower.py, test_craft_leader.py, test_craft_election.py, test_craft_stepdown.py and
test_craft_stepup.py, with their variant arguments threaded through; every output byte is compared with them, inside
canary bytes that must come back untouched.
"""
from __future__ import annotations

import ctypes as C
import random

import numpy as np
import pytest

from oracle import pyoracle as oracle
from tests import test_craft_election as te
from tests import test_craft_leader as tl
from tests import test_craft_stepdown as tsd
from tests import test_craft_stepup as ts
from tests import test_follower as tf

vi, framed = tf.vi, tf.framed
U32, U64 = (1 << 32) - 1, (1 << 64) - 1
MALFORMED = 0xFFFFFFFF
CANARY = 0xA5
PAD = 64
EDGES = (251, 1 << 16, 1 << 32)                  # the first value of each wider varint

# ---- variant settings: one tuple per setting, covering every variant of the path -------------------------------------
# the follower: (append_variant, reply_variant, meta_variant, log_variant); reply_variant stops at 250
FOLLOWER = {
    "defaults": (0, 1, 0, 1),
    "all_250": (250, 250, 250, 250),
    "all_251_up": (251, 250, 252, 253),
    "all_65535": (65535, 250, 65535, 65535),
    "log_0_rest_65535": (65535, 250, 65535, 0),
    "reply_0_rest_65535": (65535, 0, 65535, 65535),
    "reply_250_rest_3_byte": (300, 250, 1000, 4096),
}
# the leader loop: the follower's four, then the AppendEntriesReply index the leader parses (None: the follower's)
LOOP = {
    "all_250": (250, 250, 250, 250, None),
    "all_251_up": (251, 250, 252, 253, 254),
    "all_65535": (65535, 250, 65535, 65535, 65535),
    "append_0_rest_65535": (0, 250, 65535, 65535, 65534),
    "reply_250_rest_3_byte": (300, 250, 1000, 4096, None),
}
# elections: (request_vote_variant, reply_variant, the follower's meta_variant)
ELECTION = {
    "defaults": (2, 3, 0),
    "all_250": (250, 250, 250),
    "all_251_up": (251, 252, 253),
    "all_65535": (65535, 65535, 65535),
    "rv_0_rest_65535": (0, 65535, 65535),
    "mixed": (300, 3, 65535),
}
# step-down: the four PeerMsg indices (which must differ), the followers' meta_variant, log_variant and reply_variant
STEPDOWN = {
    "defaults": ((0, 1, 2, 3), 0, 1, 1),
    "all_250": ((250, 249, 248, 247), 250, 250, 249),
    "all_251_up": ((251, 252, 253, 254), 255, 256, 250),
    "all_65535": ((65535, 65534, 65533, 65532), 65535, 65535, 250),
    "ae_0_rest_65535": ((0, 65535, 65534, 65533), 65535, 65535, 250),
    "mixed": ((65535, 1, 300, 3), 0, 65535, 1),
}
# reconstruct reads, serve and absorb: (reconstruct_variant, reply_variant)
RECON = {
    "defaults": (4, 5),
    "all_250": (250, 250),
    "all_251_up": (251, 300),
    "all_65535": (65535, 65535),
    "rc_0_reply_65535": (0, 65535),
    "mixed": (65535, 5),
}


# ---- CPU: the restated encoders at every width --------------------------------------------------------------------
def test_varints_against_the_oracle():
    for v in (0, 1, 250, 251, 252, 65535, 65536, U32, 1 << 32, U64):
        assert vi(v) == oracle.varint(v)
        assert len(vi(v)) == (1 if v < 251 else 3 if v < 1 << 16 else 5 if v < 1 << 32 else 9)


def test_one_frame_of_each_kind_at_a_3_byte_variant():
    """hand-worked bytes at variant 300 (fb 2c 01)"""
    v = b"\xfb\x2c\x01"
    e = tf.entry(3, 2, 1, 3, {0: b"\xaa\xbb"}, True, 0)
    body = b"\x00" + v + bytes([4, 7, 3, 1]) + e + bytes([6, 2])
    assert tf.append_entries(4, 7, 3, [e], 6, 2, variant=300) == len(body).to_bytes(8, "big") + body
    assert tf.reply(7, 300, (6, 251), variant=300) == bytes([0] * 7 + [13, 0]) + v + bytes([7, 0xFB, 0x2C, 0x01, 1, 6, 0xFB, 0xFB, 0])
    assert tf.dur_log_entry(bytes([5, 9]), variant=300) == bytes([0] * 7 + [6]) + v + bytes([5, 9, 0])
    assert tf.dur_metadata(70000, variant=300) == bytes([0] * 7 + [9]) + v + bytes([0xFC, 0x70, 0x11, 0x01, 0x00, 0xFF])
    assert te.request_vote(5, 7, 4, variant=300) == bytes([0] * 7 + [7, 0]) + v + bytes([5, 7, 4])
    assert te.vote_reply(251, True, variant=300) == bytes([0] * 7 + [8, 0]) + v + bytes([0xFB, 0xFB, 0x00, 1])
    assert te.metadata(3, 1, variant=300) == bytes([0] * 7 + [5]) + v + bytes([3, 1])
    assert ts.reconstruct([(3, 2)], variant=300) == bytes([0] * 7 + [7, 0]) + v + bytes([1, 3, 2])
    cw = tf.codeword(3, 2, 4, {1: b"\xaa\xbb"})
    assert ts.reconstruct_reply([(7, cw)], variant=300) == framed(b"\x00" + v + bytes([1, 7]) + cw)
    assert ts.parse_reply(ts.reconstruct_reply([(7, cw)], variant=300), 3, 5, 300) == [(7, 4, {1: b"\xaa\xbb"})]
    assert ts.parse_reply(ts.reconstruct_reply([(7, cw)], variant=300), 3, 5, 5) is None
    kind, f = tf._parse_reply_py(tf.reply(7, 300, (6, 251), variant=300), 300)
    assert kind is None and f == (7, 300, (6, 251))
    assert tf._parse_reply_py(tf.reply(7, 300, variant=300), 1)[0] == 300        # another PeerMsg: its index


@pytest.mark.parametrize("v", [0, 250, 251, 65535])
def test_encoders_shift_by_the_variant_width(v):
    """each frame at variant v is the variant-0 frame with the variant's varint in its place and the length adjusted"""
    w = len(vi(v)) - 1
    e = tf.entry(1 << 32, 3, 2, 251, {4: bytes(84)}, False, 65536)
    cases = [(lambda x: tf.append_entries(U32, 1 << 16, 250, [e], U64, 7, variant=x), 9),
             (lambda x: tf.reply(U64, U64, (U64, U64), variant=x), 9),
             (lambda x: tf.dur_log_entry(e[:-3], variant=x), 8),
             (lambda x: tf.dur_metadata(U64, variant=x), 8),
             (lambda x: te.request_vote(U64, U64, U64, variant=x), 9),
             (lambda x: te.vote_reply(U64, True, variant=x), 9),
             (lambda x: te.metadata(U64, 3, variant=x), 8),
             (lambda x: ts.reconstruct([(65536, U32)] * 251, variant=x), 9),
             (lambda x: ts.reconstruct_reply([(1 << 32, tf.codeword(3, 2, 1, {0: b"\x01"}))], variant=x), 9)]
    for enc, at in cases:
        a, b = enc(0), enc(v)
        assert len(b) == len(a) + w and int.from_bytes(b[:8], "big") == len(b) - 8
        assert b[at:at + 1 + w] == vi(v) and b[at + 1 + w:] == a[at + 1:]
    # the widest cells: a reply fills 47 of its 48 bytes at reply_variant 250, RequestVote 39 of 48 and a vote reply
    # 22 of 32 at a 3-byte variant, Metadata 21 of 32
    assert len(tf.reply(U64, U64, (U64, U64), variant=250)) == 47 and len(tf.reply(U64, U64, (U64, U64), variant=251)) == 49
    assert len(te.request_vote(U64, U64, U64, variant=65535)) == 39 and len(te.vote_reply(U64, True, variant=65535)) == 22
    assert len(te.metadata(U64, 0xFF, variant=65535)) == 21 and len(tf.dur_metadata(U64, variant=65535)) == 21


# ---- CPU: the refusal edges of each call ---------------------------------------------------------------------------
def _refused(lib, _lib, rc, why):
    assert rc == _lib.SS_ERR_INVALID_ARG and why in lib.ss_last_error().decode(), (rc, lib.ss_last_error(), why)


def _passed(lib, _lib, rc, why):
    """a call whose variant checks passed: it stops later (a null handle), with another message"""
    assert rc != 0 and why not in lib.ss_last_error().decode(), (rc, lib.ss_last_error(), why)


def test_follower_config_variant_edges():
    from summerset_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    why = "reply_variant must be < 251"
    for k, edge in ((4, 1 << 16), (5, 251), (6, 1 << 16), (7, 1 << 16)):
        for v, ok in ((edge - 1, True), (edge, False), (U32, False)):
            f = [_lib.SS_PROTO_CRAFT, 5, 0, 64, 0, 1, 0, 1]
            f[k] = v
            rc = lib.ss_follower_create(None, C.byref(_lib.FollowerConfig(*f)), 4, C.byref(h))
            (_passed if ok else _refused)(lib, _lib, rc, why)


def test_call_variant_edges():
    from summerset_b200 import _lib
    lib = _lib.load()
    b = [16] * 4
    for v, ok in ((65535, True), (1 << 16, False), (U32, False)):
        chk = lambda rc, why: (_passed if ok else _refused)(lib, _lib, rc, why)
        chk(lib.ss_follower_campaign(None, 16, 1, None, v, 16, 16, 16, 16, 16, 16), "2^16")
        chk(lib.ss_follower_vote(None, 16, 0, 16, 16, 16, 1, v, 3, 16, 16, 16, 16, 16, 16), "2^16")
        chk(lib.ss_follower_vote(None, 16, 0, 16, 16, 16, 1, 2, v, 16, 16, 16, 16, 16, 16), "2^16")
        chk(lib.ss_follower_tally(None, 16, 0, 16, 16, 16, 1, v, 16, 16, 16, 16, 16, None), "2^16")
        chk(lib.ss_engine_craft_reconstruct_reads(None, None, 0, 1, v, 16, 0, *b, 1, None), "2^16")
        chk(lib.ss_engine_craft_absorb(None, 16, 0, 16, 16, 16, 1, v, 16, 16), "2^16")
        chk(lib.ss_engine_craft_backoff(None, 16, 0, 16, 16, 16, 16, 1, v, 16), "2^16")
        chk(lib.ss_append_reply_parse_dev(None, 16, 0, 16, 16, 16, 16, 1, 1, v, *([16] * 7)), "2^16")
        spec = _lib.AppendPackSpec(0, v, 1, 0, 0, 0)
        chk(lib.ss_frame_append_pack_dev(None, C.byref(spec), None, 16, 0, *b, 1, 16, 16, None), "2^16")
        for k in range(4):
            vs = [0, 1, 2, 3]
            vs[k] = v
            spec = _lib.StepDownSpec(*vs)
            chk(lib.ss_engine_craft_step_down(None, 16, C.byref(spec), 16, 0, 16, 16, 16, 1, 16, 0, 16, 16, 16, 16, None), "2^16")
    # serve checks its follower first, then both variants
    fol = C.c_void_p(16)
    for rc_v, rp_v in ((1 << 16, 5), (4, 1 << 16)):
        _refused(lib, _lib, lib.ss_follower_reconstruct_serve(fol, 16, 0, 16, 16, 16, 1, rc_v, rp_v, 16, 0, 16, 16, 16, None), "2^16")


def test_reply_parse_refuses_a_variant_of_2_16():
    """a frame whose variant is 2^16 or more is malformed for every CRaft decoder, so the reply parser refuses such a
    reply_variant, as the back-off that takes the same index does (it used to decode frames carrying it as replies)"""
    from summerset_b200 import _lib
    lib = _lib.load()
    _refused(lib, _lib, lib.ss_append_reply_parse_dev(None, 16, 0, 16, 16, 16, 16, 1, 1, 1 << 16, *([16] * 7)), "reply_variant must be < 2^16")


def test_step_down_refuses_equal_variants_at_every_width():
    from summerset_b200 import _lib
    lib = _lib.load()
    for vs in ((300, 65535, 300, 7), (0, 65535, 1, 65535), (250, 251, 252, 250), (1, 1, 2, 3), (7, 8, 65534, 65534)):
        spec = _lib.StepDownSpec(*vs)
        _refused(lib, _lib, lib.ss_engine_craft_step_down(None, 16, C.byref(spec), 16, 0, 16, 16, 16, 1, 16, 0, 16, 16, 16, 16, None),
                 "must differ")
    spec = _lib.StepDownSpec(65535, 65534, 65533, 65532)
    _passed(lib, _lib, lib.ss_engine_craft_step_down(None, 16, C.byref(spec), 16, 0, 16, 16, 16, 1, 16, 0, 16, 16, 16, 16, None),
            "variants")


# ---- GPU: the follower's append -------------------------------------------------------------------------------------
def _canaried_append(fol):
    """Follower.append with every output array and cell inside canary bytes, which must come back untouched around
    them; the cells keep their canary where the call writes nothing"""
    import torch
    from summerset_b200 import _lib

    def append(buf, fo, fg, fp, store, wal, store_capacity=None, wal_capacity=None):
        n, dev = fo.numel(), buf.device
        shapes = dict(store_off=(n, torch.int64), wal_off=(n, torch.int64), wal_len=(n, torch.int64), meta=(32 * n, torch.uint8),
                      meta_len=(n, torch.int32), replies=(48 * n, torch.uint8), reply_len=(n, torch.int32), reply_dst=(n, torch.uint8),
                      trunc_slot=(n, torch.int64), verdict=(n, torch.int32), commit_lo=(fol.G, torch.int64), totals=(2, torch.int64))
        raw, out = {}, {}
        for k, (cnt, dt) in shapes.items():
            nb = cnt * torch.tensor([], dtype=dt).element_size()
            raw[k] = torch.full((nb + 2 * PAD,), CANARY, dtype=torch.uint8, device=dev)
            out[k] = raw[k][PAD:PAD + nb].view(dt)
        p = lambda k: out[k].data_ptr()
        _lib.check(fol.lib.ss_follower_append(fol.h, buf.data_ptr(), buf.numel(), fo.data_ptr(), fg.data_ptr(), fp.data_ptr(), n,
                                              store.data_ptr(), store.numel() if store_capacity is None else store_capacity,
                                              p("store_off"), wal.data_ptr(), wal.numel() if wal_capacity is None else wal_capacity,
                                              p("wal_off"), p("wal_len"), p("meta"), p("meta_len"), p("replies"), p("reply_len"),
                                              p("reply_dst"), p("trunc_slot"), p("verdict"), p("commit_lo"), p("totals")))
        torch.cuda.synchronize()
        for k, r in raw.items():
            r = r.cpu().numpy()
            assert (r[:PAD] == CANARY).all() and (r[-PAD:] == CANARY).all(), k
        out["meta"], out["replies"] = out["meta"].view(n, 32), out["replies"].view(n, 48)
        fol.last = (store, wal, out)
        return out

    return append


def _check_bytes_outside(h, o):
    """cells past their length, WAL bytes outside the records and store bytes past the batch's regions keep their
    canary (a meta cell is zero to its end when written)"""
    store, wal, _ = h.fol.last
    for i in range(len(o["verdict"])):
        ml, rl = int(o["meta_len"][i]), int(o["reply_len"][i])
        assert ((o["meta"][i] == CANARY).all() if ml == 0 else not o["meta"][i][ml:].any()), i
        assert (o["replies"][i][rl:] == CANARY).all(), (i, rl)
    wl = wal.cpu().numpy()
    inside = np.zeros(wl.size, dtype=bool)
    for i in range(len(o["verdict"])):
        at, end = int(o["wal_off"][i]), int(o["wal_off"][i]) + int(o["wal_len"][i])
        while o["wal_len"][i] and at < end:
            ln = int.from_bytes(wl[at:at + 8].tobytes(), "big")
            inside[at:at + 8 + ln] = True
            at += tl.r16(8 + ln)
        assert o["wal_len"][i] == 0 or at == end, i
    assert (wl[~inside] == CANARY).all()
    assert (store.cpu().numpy()[int(o["totals"][0]):] == CANARY).all()


def _foreign_frames(av, g, peer, me, G):
    """frames of other messages and malformed ones, against append_variant av -> (group, peer, bytes, verdict)"""
    ae = lambda v, term=9: vi(0) + vi(v) + vi(term) + vi(0) + vi(0) + vi(0) + vi(0) + vi(0)     # an empty AppendEntries
    out = [(g, peer, framed(ae(k)), k) for k in (0, 1, 7, 250, 251, 300, 65535) if k != av]      # 1- and 3-byte indices
    out += [(g, peer, framed(vi(1) + vi(4)), 0x80000001), (g, peer, framed(vi(300) + vi(0)), 0x80000000 | 300),
            (g, peer, framed(vi(65535)), 0x80000000 | 65535), (g, peer, framed(vi(1 << 16)), MALFORMED),
            (g, peer, framed(vi(0) + vi(1 << 16) + ae(0)[2:]), MALFORMED),
            (g, peer, framed(ae(av)[:-1]), MALFORMED), (g, peer, framed(ae(av) + b"\x00"), MALFORMED),
            (g, me, framed(ae(av)), MALFORMED), (G + 1, peer, framed(ae(av)), MALFORMED)]
    return out


def _harness(n, G, setting, seed, **kw):
    from tests.test_follower import Harness
    av, rv, mv, lv = FOLLOWER[setting]
    h = Harness(n, G, seed=seed, append_variant=av, reply_variant=rv, meta_variant=mv, log_variant=lv, **kw)
    h.fol.append = _canaried_append(h.fol)
    return h


@pytest.mark.gpu
@pytest.mark.parametrize("setting", list(FOLLOWER))
@pytest.mark.parametrize("n", [3, 5, 9, 17])
def test_follower_append_at_every_variant_setting(setting, n):
    h = _harness(n, 24, setting, seed=len(setting) * 100 + n, frames_per_group=5, sharded=n in (5, 17))
    av = FOLLOWER[setting][0]
    bad = _foreign_frames(av, 3, 0, h.me, h.G)
    o, _, _ = h.batch(h.take(5), bad=bad)
    _check_bytes_outside(h, o)
    assert (o["wal_len"] > 0).sum() >= h.G // 4 and (o["meta_len"] > 0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("setting", ["defaults", "all_65535", "log_0_rest_65535", "reply_250_rest_3_byte"])
@pytest.mark.parametrize("which,short", [("wal", 0), ("wal", 1), ("store", 0), ("store", 1)])
def test_follower_capacity_cut_at_every_variant_setting(setting, which, short):
    """the WAL regions the cut sums depend on log_variant's width: at the exact capacity nothing is cut, a byte short
    the last frame is"""
    h = _harness(5, 16, setting, seed=31, frames_per_group=4, sharded=True)
    o, _, (so, wo) = h.batch(h.take(4), store_short=short if which == "store" else None, wal_short=short if which == "wal" else None)
    cut = (o["verdict"].view(np.uint32) == tf.STORE_FULL) | (o["verdict"].view(np.uint32) == tf.WAL_FULL)
    assert cut.any() == bool(short)
    _check_bytes_outside(h, o)


def _install_follower(h, groups, rng):
    """follower state through its views and into the models: groups[g] = dict(start, le, ct, terms {slot: term}); every
    installed entry holds d shards of data_len 10 in a store the harness keeps"""
    import torch
    fol, d, W = h.fol, h.d, h.W
    L = -(-10 // d)
    blob, at = bytearray(), {}
    for g, gr in enumerate(groups):
        for s in gr["terms"]:
            at[(g, s)] = len(blob)
            blob += b"".join(rng.randbytes(L) + bytes(tl.pitch(L) - L) for _ in range(d))
    store = torch.tensor(np.frombuffer(bytes(blob) + bytes(64), dtype=np.uint8), device="cuda:0")
    h.stores.append(store)
    sb, base = bytes(blob), store.data_ptr()
    arr = dict(term=fol.term.cpu().numpy(), held=fol.held.cpu().numpy(), data_len=fol.data_len.cpu().numpy(),
               shard_addr=fol.shard_addr.cpu().numpy())
    for g, gr in enumerate(groups):
        m = h.models[g]
        m.start, m.le, m.ct, m.lc, m.ls, m.ldr = gr["start"], gr["le"], gr["ct"], gr["start"], 0, 0xFF
        m.log = {}
        for s, t in gr["terms"].items():
            p_ = s & (W - 1)
            a = at[(g, s)]
            m.log[s] = (t, 10, {j: sb[a + j * tl.pitch(L):a + j * tl.pitch(L) + L] for j in range(d)})
            arr["term"][g][p_], arr["held"][g][p_], arr["data_len"][g][p_] = t, (1 << d) - 1, 10
            arr["shard_addr"][g][p_] = base + a
    for k, a in arr.items():
        getattr(fol, k).copy_(torch.from_numpy(a).to("cuda:0"))
    for k, key in (("start_slot", "start"), ("log_end", "le"), ("curr_term", "ct"), ("last_commit", "start")):
        getattr(fol, k).copy_(torch.tensor([gr[key] for gr in groups], dtype=torch.int64, device="cuda:0"))
    fol.last_snap.zero_()
    fol.leader.fill_(0xFF)
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("setting", list(FOLLOWER))
def test_follower_fields_across_width_edges(setting):
    """each group's ring runs across a slot width edge (250/251, 65535/65536, 2^32 - 1/2^32) and its term across a term
    edge, both at once; a far group keeps every field at 9 bytes, which makes the widest reply.  Frames append across the
    edge, are refused with a conflict walk-back across it, raise the term across its edge and truncate there, commit
    through it and run past the window."""
    h = _harness(5, 10, setting, seed=77, frames_per_group=0)
    rng, d, n, W = h.rng, h.d, h.n, h.W
    combos = [(es, et) for es in EDGES for et in EDGES] + [(1 << 40, 1 << 40)]
    groups = []
    for es, et in combos:
        start = es - 4
        groups.append(dict(start=start, le=es - 1, ct=et - 1, terms={start: et - 2, start + 1: et - 1, start + 2: et - 1}))
    _install_follower(h, groups, rng)
    L = -(-10 // d)
    ent = lambda t, lo: tf.Ent(t, d, n - d, 10, {j: rng.randbytes(L) for j in range(d)}, rng.random() < 0.5, lo)
    frames = []
    for g, ((es, et), gr) in enumerate(zip(combos, groups)):
        pe = g % (n - 1)
        lo = rng.choice(EDGES) - rng.randint(0, 1)                            # log_offset, dropped from the record
        frames += [(g, (pe, et - 1, es - 2, et - 1, [ent(et - 1, lo) for _ in range(4)], es + 5, es)),  # slots es-1 .. es+2
                   (g, (pe, et - 1, es + 2, et, [], 0, 0)),                                       # conflict: walks back to start + 1
                   (g, (pe, et, es - 1, et - 1, [ent(et, lo) for _ in range(2)], 0, 0)),          # raise, truncate at es
                   (g, (pe, et, es + 1, et, [], es + 1, es + 1)),                                 # commit through the edge
                   (g, (pe, et, es + W, et, [ent(et, 0)], 0, 0))]                                 # past the window
    o, seq, _ = h.batch(frames)
    _check_bytes_outside(h, o)
    v = o["verdict"].view(np.uint32)
    assert (v == tf.REJECTED).sum() == len(combos) and (v == tf.BEYOND).sum() == len(combos)
    assert int((o["trunc_slot"] != -1).sum()) == len(combos)
    widest = max(int(x) for x in o["reply_len"])
    assert widest == len(tf.reply(U64, U64, (U64, U64), variant=FOLLOWER[setting][1]))
    assert [m.lc for m in h.models] == [es + 1 for es, _ in combos]
    assert [m.ct for m in h.models] == [et for _, et in combos]


# ---- GPU: the leader's pack, the follower, the reply parser and the back-off ----------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("setting", list(LOOP))
def test_leader_loop_at_every_variant_setting(setting):
    av, rv, mv, lv, lrv = LOOP[setting]
    tl.closed_loop(9 if setting == "all_65535" else 5, av, rv, mv, lv, lrv)


def _reply_parse_raw(ctx, buf, offs, grp, peer, curr_term, G, rv):
    import torch
    from summerset_b200 import _lib
    n = len(offs)
    shapes = dict(rec_group=torch.int32, rec_peer=torch.uint8, rec_end_slot=torch.int32, rec_term=torch.int64,
                  rec_conflict_term=torch.int64, rec_conflict_slot=torch.int64, rec_kind=torch.int32)
    raw, out = {}, {}
    for k, dt in shapes.items():
        nb = n * torch.tensor([], dtype=dt).element_size()
        raw[k] = torch.full((nb + 2 * PAD,), CANARY, dtype=torch.uint8, device="cuda:0")
        out[k] = raw[k][PAD:PAD + nb].view(dt)
    t = lambda a, dt: torch.tensor(a, dtype=dt, device="cuda:0")
    tb, fo, fg, fp = buf, t(offs, torch.int64), t(np.array(grp, dtype=np.uint32).view(np.int32), torch.int32), t(peer, torch.uint8)
    p = lambda k: out[k].data_ptr()
    _lib.check(ctx.lib.ss_append_reply_parse_dev(ctx.h, tb.data_ptr(), tb.numel(), fo.data_ptr(), fg.data_ptr(), fp.data_ptr(),
                                                 curr_term.data_ptr(), n, G, rv, *(p(k) for k in shapes)))
    torch.cuda.synchronize()
    for k, r in raw.items():
        r = r.cpu().numpy()
        assert (r[:PAD] == CANARY).all() and (r[-PAD:] == CANARY).all(), k
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("rv", [0, 1, 250, 251, 300, 65535])
def test_reply_parse_at_every_variant_and_field_width(rv):
    """AppendEntriesReply frames at reply_variant rv, which a leader can receive at any index below 2^16: terms at and
    around each edge against the engine's u32 curr_term, end_slot on both sides of 2^32 (END_RANGE), conflict fields of
    every width, other messages of both widths and malformed frames"""
    import torch
    from summerset_b200.engine import RaftEngine
    ctx = ts._ctx()
    G = 6
    eng = RaftEngine(ctx, G, 5, craft=True)
    cts = [5, 250, 251, 65535, 65536, U32]
    eng.curr_term.copy_(torch.tensor(np.array(cts, dtype=np.uint32).view(np.int32), device="cuda:0"))
    rng = random.Random(rv)
    frames = []
    for g, ct in enumerate(cts):
        for end in (0, 250, 251, 65535, 65536, U32, 1 << 32, U64):
            frames.append((g, rng.randrange(4), tf.reply(ct, end, None, rv)))
        for c in ((250, 251), (65535, 65536), (U32, 1 << 32), (U64, U64)):
            frames.append((g, rng.randrange(4), tf.reply(ct - 1, 1 << 16, c, rv)))
        frames += [(g, 0, tf.reply(ct + 1, 3, None, rv)), (g, 1, tf.reply(U64, U64, (U64, U64), rv))]
        frames += [(g, 2, tf.reply(ct, 3, None, k)) for k in (0, 1, 2, 250, 251, 65534, 65535) if k != rv]
        ok = tf.reply(ct, 3, None, rv)
        frames += [(g, 3, framed(ok[8:-1])), (g, 3, framed(ok[8:] + b"\x00")), (g, 3, framed(ok[8:-1] + b"\x02")),
                   (g, 0, framed(vi(1) + vi(2))), (g, 0, framed(vi(300))), (g, 0, framed(vi(1 << 16))),
                   (g, 0, framed(vi(0) + vi(1 << 16) + ok[8 + 1 + len(vi(rv)):]))]
    frames.append((G, 0, tf.reply(1, 1, None, rv)))
    buf, offs = ts._buf([x for _, _, x in frames], rng)
    r = _reply_parse_raw(ctx, buf, offs, [f[0] for f in frames], [f[1] for f in frames], eng.curr_term, G, rv)
    kinds = set()
    for k, (g, pe, fr) in enumerate(frames):
        kind, f = tf._parse_reply_py(fr, rv)
        if kind is None and g >= G:
            kind, f = MALFORMED, None
        if kind is None:
            tm, end, conf = f
            kind = tf.HIGHER if tm > cts[g] else tf.CONFLICT if conf else tf.END_RANGE if end >= 1 << 32 else tf.INGEST
        else:
            tm = end = 0
            conf = None
        kinds.add(kind)
        assert int(r["rec_kind"].view(np.uint32)[k]) == kind, (k, hex(int(r["rec_kind"].view(np.uint32)[k])), hex(kind))
        assert int(r["rec_term"][k]) & U64 == tm and int(r["rec_conflict_term"][k]) & U64 == (conf[0] if conf else 0)
        assert int(r["rec_conflict_slot"][k]) & U64 == (conf[1] if conf else 0)
        ing = kind == tf.INGEST
        assert int(r["rec_group"].view(np.uint32)[k]) == (g if ing else U32) and int(r["rec_peer"][k]) == (pe if ing else 0xFF)
        assert int(r["rec_end_slot"].view(np.uint32)[k]) == (end if ing else 0)
    assert {tf.INGEST, tf.CONFLICT, tf.HIGHER, tf.END_RANGE, MALFORMED, 0x80000001, 0x80000000 | 300} <= kinds
    eng.close()


# ---- GPU: elections -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("setting", list(ELECTION))
def test_elections_at_every_variant_setting(setting):
    """campaigns, votes and tallies at the setting's RequestVote, RequestVoteReply and Metadata indices, over the rig's
    curr_terms at every width; then the widest RequestVote a follower takes (39 bytes at a 3-byte variant), its
    22-byte reply, and a campaign whose last slot and term are 9-byte varints"""
    import torch
    rvv, rpv, mv = ELECTION[setting]
    rig = te._Rig(5, 48, seed=7300 + len(setting), request_vote_variant=rvv, reply_variant=rpv, meta_variant=mv)
    for _ in range(2):
        te._round(rig, 2 * rig.G, 3 * rig.G)
    other = (rig.me + 1) % rig.n
    big = (1 << 63) - 1                                                # a 9-byte varint the int64 views hold
    rig.vote([(0, other, te.request_vote(big, big, big, rvv), (big, big, big)),
              (1, other, te.request_vote(1 << 32, 65536, 251, rvv), (1 << 32, 65536, 251))])
    # a campaign from a log that ends at slot 2^63 - 2 with a last term of 2^64 - 1
    g = 2
    nd = rig.nodes[g]
    le = (1 << 63) - 1
    nd.log, nd.le, nd.ct, nd.ldr = {le - 1: (U64, 0, {})}, le, U32 - 1, te.NONE
    rig.fol.log_end[g] = le
    rig.fol.curr_term[g] = U32 - 1
    rig.fol.leader[g] = te.NONE
    rig.fol.term[g][(le - 1) & (rig.W - 1)] = -1
    torch.cuda.synchronize()
    want = rig.campaign([g], None)
    assert want[0][0] == te.DONE and len(want[0][2]) == 8 + 1 + len(vi(rvv)) + 5 + 9 + 9
    rig.fol.close()


# ---- GPU: step-down -------------------------------------------------------------------------------------------------
def _malformed(spec, kind, term):
    ae, aer, rv, rvr = spec
    return {0: framed(vi(0) + vi(ae) + vi(term) + vi(0)), 1: framed(vi(0) + vi(aer) + vi(term) + vi(1)),
            2: framed(vi(0) + vi(rv) + vi(term) + vi(1)), 3: framed(vi(0) + vi(rvr) + vi(term) + bytes([2]))}[kind]


@pytest.mark.gpu
@pytest.mark.parametrize("setting", list(STEPDOWN))
def test_step_down_at_every_variant_setting(setting):
    """each group is deposed by one kind of message at a term on either side of each width edge, after malformed frames
    of the four indices, a RANGE term (2^32) and messages of other indices; the Metadata cell each deposing frame
    writes is the follower's meta_variant and the new term"""
    import torch
    spec, mv, lv, frv = STEPDOWN[setting]
    ae, aer, rv, rvr = spec
    n = 5
    rig = tsd._PlainRig(n, append_variant=ae, reply_variant=frv, meta_variant=mv, log_variant=lv)
    G = rig.G
    before = rig.snapshot()
    terms = [250, 251, 65535, 65536, U32]
    big = (1 << 32) - 2
    others = [k for k in (4, 5, 251, 65531) if k not in spec]
    frames, model, tt, i_of = [], [], {}, {}
    for g in range(G):
        kind, t = g % 4, terms[(g // 4 + g) % len(terms)]
        tt[g] = t
        for k in range(4):
            frames.append((g, 1 + k % (n - 1), _malformed(spec, k, big)))
            model.append((g, MALFORMED, 0))
        for k in others:
            frames.append((g, 2, framed(vi(0) + vi(k) + vi(big))))
            model.append((g, "pass", 0))
        frames += [(g, 3, framed(vi(1) + vi(0))), (g, 3, framed(vi(300)))]
        model += [(g, 0x80000001, 0), (g, 0x80000000 | 300, 0)]
        if g % 3 == 0:
            frames.append((g, 2, te.request_vote(1 << 32, 0, 0, rv)))
            model.append((g, "term", 1 << 32))
        x = {0: lambda: tf.append_entries(t, 0, 0, [], 0, 0, ae), 1: lambda: tf.reply(t, 1, None, aer),
             2: lambda: te.request_vote(t, 0, 0, rv), 3: lambda: te.vote_reply(t, False, rvr)}[kind]()
        i_of[g] = len(frames)
        frames.append((g, 1, x))
        model.append((g, "term", t))
        frames.append((g, 2, te.vote_reply(big, True, rvr)))
        model.append((g, "term", big))
    want, deposed = tsd.check_term_batch(model, {g: 1 for g in range(G)}, {g: 1 for g in range(G)})
    assert deposed == tt
    buf, fo, fg, fp = tsd._frames(frames, rig.rng)
    store = torch.zeros(1 << 23, dtype=torch.uint8, device="cuda:0")
    res = tsd._step_down_raw(rig.eng, rig.fols[0], buf, fo, fg, fp, store, variants=spec)
    assert res["verdict"].cpu().numpy().view(np.uint32).tolist() == want
    tsd._check_deposed(rig, before, range(G), tt, 1, store, res, i_of, held_all=True)
    ml = res["meta_len"].cpu().numpy()
    assert all(ml[i] == 0 for i in range(len(frames)) if i not in i_of.values())


# ---- GPU: reconstruct reads, serve and absorb ---------------------------------------------------------------------
def _recon_round(eng, peer, fs, fp, store, rv_, keep, rng, rcv, rpv, chunk, groups=None):
    """reads from the engine, served by `peer`, absorbed back, every byte against the restatements -> frames served"""
    import torch
    G, W, T = eng.G, eng.W, eng.P + 1
    d = T // 2 + 1
    out = torch.full((1 << 20,), CANARY, dtype=torch.uint8, device="cuda:0")
    lgs = [dict(last_exec=f["last_exec"], start=f["start"], last_recon=int(rv_["last_recon"][g]), lc=f["lc"], held=dict(f["held"]),
                term=f["term"]) for g, f in enumerate(fs)]
    listed = [ts.recon_walk(lg, d) for lg in lgs]
    r = eng.reconstruct_reads(out, 4096, chunk, reconstruct_variant=rcv)
    torch.cuda.synchronize()
    want = [(g, x) for g in range(G) for x in ts.recon_frames(listed[g], chunk, rcv)]
    asked = [(g, listed[g][k:k + chunk]) for g in range(G) for k in range(0, len(listed[g]), chunk)]
    nf = int(r["totals"][0])
    assert nf == len(want)
    on = out.cpu().numpy()
    inside = np.zeros(on.size, dtype=bool)
    for k, (g, x) in enumerate(want):
        off = int(r["frame_off"][k])
        assert (int(r["frame_group"][k]), int(r["frame_dst"][k]), int(r["frame_len"][k])) == (g, 0xFF, len(x))
        assert on[off:off + len(x)].tobytes() == x
        inside[off:off + ts.r16(len(x))] = True                        # the region's pad is the call's
    assert (on[~inside] == CANARY).all()
    assert rv_["last_recon"].cpu().tolist() == [lg["last_recon"] for lg in lgs]
    # serve them, and a foreign index of each width, a PeerMessage variant and a truncated frame
    reqs = [x for _, x in want]
    foreign = [k for k in (4, 5, 300) if k != rcv][0]
    extra = [ts.reconstruct([(1, 1)], variant=foreign), framed(vi(2)), framed(ts.reconstruct([(1, 1)], rcv)[8:-1])]
    grp = [g for g, _ in want] + [0, 0, 0]
    buf, offs = ts._buf(reqs + extra, rng)
    rout = torch.full((1 << 22,), CANARY, dtype=torch.uint8, device="cuda:0")
    s_ = peer.reconstruct_serve(buf, ts._t(offs, torch.int64), ts._t(grp, torch.int32), ts._t([0] * len(grp), torch.uint8), rout,
                                reconstruct_variant=rcv, reply_variant=rpv)
    torch.cuda.synchronize()
    ro = rout.cpu().numpy()
    pstore, pbase = keep[1].cpu().numpy(), keep[1].data_ptr()

    def pshard(g, s, j):
        L = -(-fp[g]["dl"][s] // d)
        at = fp[g]["addr"][s] - pbase + ts.popc(fp[g]["held"][s] & ((1 << j) - 1)) * ts.pitch(L)
        return pstore[at:at + L].tobytes()

    replies, inside = [], np.zeros(ro.size, dtype=bool)
    for i, (g, sl) in enumerate(asked):
        w = ts.serve(fp[g], sl, d, T, lambda s, j: pshard(g, s, j), rpv)
        assert int(s_["verdict"][i]) & U32 == ts.ACCEPTED
        if w is None:
            assert int(s_["reply_len"][i]) == 0
            continue
        off = int(s_["reply_off"][i])
        assert int(s_["reply_len"][i]) == len(w) and ro[off:off + len(w)].tobytes() == w, i
        inside[off:off + ts.r16(len(w))] = True
        replies.append((g, w))
    assert (ro[~inside] == CANARY).all()
    assert [int(x) & U32 for x in s_["verdict"][len(want):].cpu().tolist()] == [foreign, 0x80000002, MALFORMED]
    # absorb at reply_variant rpv, with a reply at another index that must absorb nothing
    pool = replies + [(replies[0][0], ts.reconstruct_reply([], variant=[k for k in (5, 6, 65534) if k != rpv][0]))]
    lgs2 = [dict(start=f["start"], le=f["le"], dl=dict(f["dl"]), held=dict(f["held"]), plane={}) for f in fs]
    want_abs = [None] * len(pool)
    for g in range(G):
        idx = [i for i, (h, _) in enumerate(pool) if h == g]
        for i, a in zip(idx, ts.absorb(lgs2[g], [pool[i][1] for i in idx], d, T, rpv)):
            want_abs[i] = a
    buf, offs = ts._buf([x for _, x in pool], rng)
    a = eng.absorb(buf, ts._t(offs, torch.int64), ts._t([g for g, _ in pool], torch.int32), ts._t([1] * len(pool), torch.uint8), rpv)
    torch.cuda.synchronize()
    for i, w in enumerate(want_abs):
        ver = int(a["verdict"][i]) & U32
        assert (ver == ts.ACCEPTED and int(a["absorbed"][i]) == w) if w is not None else (ver != ts.ACCEPTED and int(a["absorbed"][i]) == 0), i
    held, addr = rv_["held"].cpu().numpy(), eng.log_view()["shard_addr"].cpu().numpy()
    planes, sbase = store.cpu().numpy(), store.data_ptr()
    for g in range(G):
        for s in range(lgs2[g]["start"], lgs2[g]["le"]):
            assert int(held[g][s & (W - 1)]) & U32 == lgs2[g]["held"][s], (g, s)
        for (s, j), x in lgs2[g]["plane"].items():
            o_ = int(addr[g][s & (W - 1)]) - sbase
            got = planes[j][o_:o_ + ts.r16(len(x))].tobytes()
            assert got[:len(x)] == x and not any(got[len(x):])
    return len(want)


@pytest.mark.gpu
@pytest.mark.parametrize("setting", list(RECON))
def test_reconstruct_at_every_variant_setting(setting):
    rcv, rpv = RECON[setting]
    ctx, eng, src, peer, store, shards, fs, fp, keep, rng = ts._serve_absorb_case(5, 900 + len(setting))
    assert _recon_round(eng, peer, fs, fp, store, eng.recon_view(), keep, rng, rcv, rpv, 3) > 0
    for o in (eng, src, peer):
        o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("setting", ["defaults", "all_65535", "rc_0_reply_65535"])
def test_reconstruct_entry_counts_and_slots_across_width_edges(setting):
    """one group's log of 260 entries from slot 65400, so that a single Reconstruct and its ReconstructReply carry a
    3-byte entry count and slots on both sides of 2^16; a second group's log starts at 240 and crosses 250/251"""
    import torch
    from summerset_b200.engine import Follower, RaftEngine
    rcv, rpv = RECON[setting]
    ctx = ts._ctx()
    n, G, W = 5, 2, 512
    d, T = n // 2 + 1, n
    rng = random.Random(4242)
    src, peer = Follower(ctx, G, n, 1, window=W), Follower(ctx, G, n, 2, window=W)
    base, pgroups = [], []
    for g, (start, span) in enumerate(((65400, 260), (240, 20))):
        ent, pent = {}, {}
        for s in range(start, start + span):
            b = rng.randbytes(rng.choice((1, 7, 40)))
            ent[s] = (1 + (s - start) // 100, b, 1 << rng.randrange(T))
            pent[s] = (ent[s][0], b, (1 << T) - 1 - ent[s][2])
        le = start + span
        base.append(dict(start=start, le=le, ct=9, lc=le - 1, ls=start, last_exec=start - 1, ent=ent))
        pgroups.append(dict(start=start, le=le, ct=9, lc=start - 1, ls=start, last_exec=start - 1, ent=pent))
    st1, _ = ts._install(src, base, rng)
    st2, _ = ts._install(peer, pgroups, rng)
    eng = RaftEngine(ctx, G, n, craft=True, window=W)
    store = torch.zeros((T, 1 << 16), dtype=torch.uint8, device="cuda:0")
    o = eng.step_up(src, ts._t(list(range(G)), torch.int32), ts._t([9] * G, torch.int64), store)
    torch.cuda.synchronize()
    assert o["verdict"].cpu().tolist() == [ts.DONE] * G
    fs, fp = ts._fol_state(src), ts._fol_state(peer)
    assert _recon_round(eng, peer, fs, fp, store, eng.recon_view(), [st1, st2], rng, rcv, rpv, 300) == G
    for x in (eng, src, peer):
        x.close()
