"""CRaft leader fail-over on the device: ss_engine_craft_step_up, ss_engine_craft_reconstruct_reads,
ss_follower_reconstruct_serve and ss_engine_craft_absorb, and the held mask they give the leader's log.

The restatements below follow the reference message by message: `step_up` is the log half of become_the_leader
(craft/leadership.rs:212-246), `recon_walk` the recon half of handle_msg_append_entries_reply's success branch
(craft/messages.rs:316-371), `serve` handle_msg_reconstruct (:621-662) and `absorb` handle_msg_reconstruct_reply
(:664-744) without its execution loop.  The bincode encoders and the follower / leader restatements come from
tests/test_follower.py and tests/test_craft_leader.py.  GPU tests compare every engine word, ring entry and plane byte
with the restatements, and run a leader crash end to end: the payloads the new leader executes must be the original
request batches.
"""
from __future__ import annotations

import ctypes as C
import random

import numpy as np
import pytest

from oracle import pyoracle as oracle
from tests import test_craft_leader as tl
from tests import test_follower as tf

vi, framed = tf.vi, tf.framed
pitch, r16 = tl.pitch, tl.r16
popc = lambda x: bin(x).count("1")
U32 = (1 << 32) - 1
DONE, IGNORED, WINDOW, RANGE, STALE, STORE_FULL = range(6)
ACCEPTED, MALFORMED, OUT_FULL = 0xFFFFFFF0, 0xFFFFFFFF, 0xFFFFFFF8
STATUS_FRAME_OVERFLOW, STATUS_STORE_FULL = 4, 16


# ---- bincode ------------------------------------------------------------------------------------------------------
def reconstruct(slots, variant=4) -> bytes:
    """PeerMessage::Msg{Reconstruct{slots: Vec<(usize, Term)>}} behind its length"""
    return framed(vi(0) + vi(variant) + vi(len(slots)) + b"".join(vi(s) + vi(t) for s, t in slots))


def reconstruct_reply(entries, variant=5) -> bytes:
    """PeerMessage::Msg{ReconstructReply{slots_data: HashMap<usize, RSCodeword>}}; entries [(slot, codeword bytes)] in
    wire order"""
    return framed(vi(0) + vi(variant) + vi(len(entries)) + b"".join(vi(s) + cw for s, cw in entries))


def codeword_wide(d: int, p: int, data_len: int, shards: dict, tags) -> bytes:
    """an RSCodeword whose k-th present shard has its length as the non-minimal varint of tag tags[k % len(tags)]
    (251: 2 bytes, 252: 4, 253: 8)"""
    L = -(-data_len // d)
    out = bytes([d, p]) + vi(data_len) + vi(L) + vi(d + p)
    k = 0
    for j in range(d + p):
        if j in shards:
            t = tags[k % len(tags)]
            out += b"\x01" + bytes([t]) + L.to_bytes({251: 2, 252: 4, 253: 8}[t], "little") + shards[j]
            k += 1
        else:
            out += b"\x00"
    return out + b"\x00"


def with_data_copy(cw: bytes, data: bytes) -> bytes:
    """the codeword with data_copy Some(data) instead of None"""
    assert cw[-1] == 0
    return cw[:-1] + b"\x01" + data


def rvi(b: bytes, n: int):
    t = b[n]
    if t < 251:
        return t, n + 1
    k = {251: 2, 252: 4, 253: 8}[t]
    return int.from_bytes(b[n + 1:n + 1 + k], "little"), n + 1 + k


def parse_reply(fr: bytes, d: int, T: int, variant=5):
    """-> [(slot, data_len, {j: shard})] in wire order, or None when malformed (ss_acceptor_absorb's rules)"""
    try:
        ln = int.from_bytes(fr[:8], "big")
        b = fr[8:8 + ln]
        if len(b) != ln:
            return None
        v, n = rvi(b, 0)
        w, n = rvi(b, n)
        if v != 0 or w != variant:
            return None
        cnt, n = rvi(b, n)
        out = []
        for _ in range(cnt):
            slot, n = rvi(b, n)
            if b[n] != d or b[n + 1] != T - d:
                return None
            n += 2
            dl, n = rvi(b, n)
            L, n = rvi(b, n)
            k, n = rvi(b, n)
            if dl > U32 or k != T or L != -(-dl // d):
                return None
            sh = {}
            for j in range(T):
                tag = b[n]
                n += 1
                if tag == 1:
                    x, n = rvi(b, n)
                    if x != L or len(b) - n < L:
                        return None
                    sh[j] = bytes(b[n:n + L])
                    n += L
                elif tag != 0:
                    return None
            tag = b[n]
            n += 1
            if tag == 1:
                if len(b) - n < dl:
                    return None
                n += dl
            elif tag != 0:
                return None
            out.append((slot, dl, sh))
        return out if n == ln else None
    except IndexError:
        return None


# ---- the restatements ---------------------------------------------------------------------------------------------
def stepup_verdict(fg, W, term):
    """fg: one follower group, dict(start, le, ct, ls, term={slot: term}) -> its verdict (the checks in order)"""
    if fg["le"] - fg["start"] > W:
        return WINDOW
    if fg["le"] > U32 or term > U32 or fg["ls"] > U32 or any(fg["term"][s] > U32 for s in range(fg["start"], fg["le"])):
        return RANGE
    if term < fg["ct"]:
        return STALE
    return DONE


def step_up(fols, listing, terms, W, d, stride, G):
    """fols[g]: dict(start, le, ct, lc, ls, last_exec, term, dl, held); -> (verdicts, shard_off (None: not stepped up),
    need, {g: {slot: plane offset}})"""
    first, verdicts, sizes = {}, [], []
    for i, g in enumerate(listing):
        if g >= G or g in first:
            verdicts.append(IGNORED)
            sizes.append(0)
            continue
        first[g] = i
        v = stepup_verdict(fols[g], W, terms[i])
        verdicts.append(v)
        fg = fols[g]
        sizes.append(sum(pitch(-(-fg["dl"][s] // d)) for s in range(fg["start"], fg["le"]) if fg["dl"][s]) if v == DONE else 0)
    offs, at = [], 0
    for x in sizes:
        offs.append(at)
        at += x
    need, slots, out = at, {}, []
    for i, g in enumerate(listing):
        if verdicts[i] == DONE and offs[i] + sizes[i] > stride:
            verdicts[i] = STORE_FULL
        if verdicts[i] != DONE:
            out.append(None)
            continue
        out.append(offs[i])
        fg, o, slots[g] = fols[g], offs[i], {}
        for s in range(fg["start"], fg["le"]):
            if fg["dl"][s]:
                slots[g][s] = o
                o += pitch(-(-fg["dl"][s] // d))
    return verdicts, out, need, slots


def recon_walk(lg, d):
    """lg: dict(last_exec, start, last_recon, lc, held={s}, term={s}) -> the (slot, term) listed; moves last_recon"""
    out = []
    for s in range(max(lg["last_exec"] + 1, lg["start"], lg["last_recon"] + 1), lg["lc"] + 1):
        if popc(lg["held"][s]) < d:
            out.append((s, lg["term"][s]))
    if out:
        lg["last_recon"] = out[-1][0]
    return out


def recon_frames(listed, chunk, variant=4):
    return [reconstruct(listed[k:k + chunk], variant) for k in range(0, len(listed), chunk)]


def serve(fg, slots, d, T, shard, variant=5):
    """fg: dict(start, le, term, dl, held); shard(s, j) -> bytes; the ReconstructReply bytes, or None (empty map)"""
    seen, ents = set(), []
    for s, t in slots:
        if s < fg["start"] or s >= fg["le"] or fg["term"][s] != t or (s, t) in seen:
            continue
        seen.add((s, t))
        ents.append((s, tf.codeword(d, T - d, fg["dl"][s], {j: shard(s, j) for j in range(T) if fg["held"][s] >> j & 1})))
    return reconstruct_reply(ents, variant) if ents else None


def absorb(lg, frames, d, T, variant=5):
    """lg: dict(start, le, dl={s}, held={s}, plane={(s, j): bytes}); frames: the group's frame bytes in frame order ->
    absorbed per frame (None: malformed)"""
    res = []
    for fr in frames:
        ents = parse_reply(fr, d, T, variant)
        if ents is None:
            res.append(None)
            continue
        taken = 0
        for k, (s, dl, sh) in enumerate(ents):
            if any(x[0] == s for x in ents[k + 1:]):                 # a HashMap decode keeps the last insert
                continue
            if s < lg["start"] or s >= lg["le"] or not lg["dl"].get(s) or dl != lg["dl"][s]:
                continue
            add = [j for j in sh if not lg["held"][s] >> j & 1]
            if not add:
                continue
            for j in add:
                lg["plane"][(s, j)] = sh[j]
                lg["held"][s] |= 1 << j
            taken += 1
        res.append(taken)
    return res


# ---- CPU: hand-worked cases ---------------------------------------------------------------------------------------
def test_reconstruct_bytes():
    # length 8 bytes, Msg 0, variant 4, two entries: (3, term 2) and (300, term 70000)
    want = bytes.fromhex("000000000000000d" "00" "04" "02" "03" "02" "fb2c01" "fc70110100")
    assert reconstruct([(3, 2), (300, 70000)]) == want
    assert reconstruct([]) == bytes.fromhex("0000000000000003000400")


def test_reconstruct_reply_bytes_with_data_copy_and_a_repeated_key():
    # RS(3,2), data_len 4, shard_len 2: slot 7 carries shard 1 with data_copy Some, slot 7 again carries shard 4
    cw1 = with_data_copy(tf.codeword(3, 2, 4, {1: b"\xaa\xbb"}), b"\x01\x02\x03\x04")
    cw2 = tf.codeword(3, 2, 4, {4: b"\xcc\xdd"})
    assert cw1 == bytes.fromhex("03 02 04 02 05 00 01 02aabb 00 00 00 01 01020304".replace(" ", ""))
    assert cw2 == bytes.fromhex("03 02 04 02 05 00 00 00 00 01 02ccdd 00".replace(" ", ""))
    fr = reconstruct_reply([(7, cw1), (7, cw2)])
    assert fr[8:11] == b"\x00\x05\x02" and len(fr) == 8 + 3 + 2 * 1 + len(cw1) + len(cw2)
    assert parse_reply(fr, 3, 5) == [(7, 4, {1: b"\xaa\xbb"}), (7, 4, {4: b"\xcc\xdd"})]
    lg = dict(start=5, le=9, dl={7: 4}, held={7: 0b00001}, plane={})
    assert absorb(lg, [fr], 3, 5) == [1]                          # the repeated key keeps its last value only
    assert lg["held"][7] == 0b10001 and lg["plane"] == {(7, 4): b"\xcc\xdd"}


def test_encoders_match_the_oracle():
    for v in (0, 250, 251, 65535, 65536, U32, 1 << 32):
        assert vi(v) == oracle.varint(v)
    for d, p, dl in ((2, 1, 3), (3, 2, 4096), (7, 6, 250)):
        L = -(-dl // d)
        rng = np.random.default_rng(dl)
        sh = {j: rng.integers(0, 256, L, dtype=np.uint8).tobytes() for j in range(d + p) if j % 3 == 1}
        wal = oracle.wal_accept_data(0, 0, d, p, dl, [sh.get(j) for j in range(d + p)])
        assert reconstruct_reply([(0, tf.codeword(d, p, dl, sh))])[12:] == wal[8 + 3:]   # AcceptData 1, slot 0, ballot 0


def test_model_recon_walk_and_last_recon():
    lg = dict(last_exec=2, start=1, last_recon=0, lc=8, held={s: 0b1 if s % 2 else 0b111 for s in range(1, 10)},
              term={s: 1 + s // 5 for s in range(1, 10)})
    assert recon_walk(lg, 3) == [(3, 1), (5, 2), (7, 2)] and lg["last_recon"] == 7
    assert recon_walk(lg, 3) == []                                # listed already
    lg["lc"] = 9
    assert recon_walk(lg, 3) == [(9, 2)] and lg["last_recon"] == 9
    assert [len(f) for f in recon_frames([(3, 1), (5, 2), (7, 2)], 2)] == [8 + 3 + 4, 8 + 3 + 2]


def test_model_serve_skips_and_repeats():
    fg = dict(start=4, le=8, term={s: 3 for s in range(4, 8)}, dl={s: 10 for s in range(4, 8)}, held={s: 0b00100 for s in range(4, 8)})
    shard = lambda s, j: bytes([s]) * 4
    assert serve(fg, [(3, 3), (8, 3), (5, 2)], 3, 5, shard) is None   # below start, at log_end, another term
    got = serve(fg, [(6, 3), (5, 3), (6, 3)], 3, 5, shard)
    assert got == reconstruct_reply([(6, tf.codeword(3, 2, 10, {2: b"\x06" * 4})), (5, tf.codeword(3, 2, 10, {2: b"\x05" * 4}))])


def test_model_step_up_verdicts_and_offsets():
    def fg(start, le, ct=1, t=1, dl=100):
        return dict(start=start, le=le, ct=ct, lc=le - 1, ls=0, last_exec=0, term={s: t for s in range(start, le)},
                    dl={s: dl if s else 0 for s in range(start, le)}, held={s: 1 for s in range(start, le)})
    fols = [fg(0, 4), fg(0, 70), fg(2, 5, t=1 << 32), fg(1, 3, ct=9), fg(0, 3)]
    v, off, need, slots = step_up(fols, [0, 1, 2, 3, 4, 0, 7], [2, 2, 2, 2, 2, 2, 2], 64, 3, 10 ** 6, 5)
    assert v == [DONE, WINDOW, RANGE, STALE, DONE, IGNORED, IGNORED]
    assert off == [0, None, None, None, 3 * 64, None, None] and need == 5 * 64 and slots[4] == {1: 192, 2: 256}
    v, off, _, _ = step_up(fols, [0, 4], [2, 2], 64, 3, 5 * 64 - 1, 5)
    assert v == [DONE, STORE_FULL]                                # a suffix is cut by the plane stride


def test_non_minimal_shard_lengths_decode():
    # RS(3,2), data_len 6, shard_len 2: shard 1's length as fb 02 00, shard 3's as fc 02 00 00 00
    cw = codeword_wide(3, 2, 6, {1: b"\x11\x22", 3: b"\x33\x44"}, (251, 252))
    assert cw == bytes.fromhex("03 02 06 02 05 00 01fb0200 1122 00 01fc02000000 3344 00 00".replace(" ", ""))
    lg = dict(start=1, le=3, dl={2: 6}, held={2: 0b00001}, plane={})
    assert absorb(lg, [reconstruct_reply([(2, cw)])], 3, 5) == [1]
    assert lg["plane"] == {(2, 1): b"\x11\x22", (2, 3): b"\x33\x44"} and lg["held"][2] == 0b01011


def test_model_absorb_first_carrier_wins_and_filters():
    lg = dict(start=2, le=6, dl={2: 0, 3: 9, 4: 9, 5: 9}, held={2: 0, 3: 0b001, 4: 0b111, 5: 0}, plane={})
    a = reconstruct_reply([(3, tf.codeword(3, 2, 9, {1: b"A" * 3})), (4, tf.codeword(3, 2, 9, {3: b"B" * 3}))])
    b = reconstruct_reply([(3, tf.codeword(3, 2, 9, {1: b"C" * 3, 2: b"D" * 3})), (5, tf.codeword(3, 2, 8, {0: b"E" * 3})),
                           (6, tf.codeword(3, 2, 9, {0: b"F" * 3})), (2, tf.codeword(3, 2, 9, {0: b"G" * 3}))])
    assert absorb(lg, [a, b, a[:-1]], 3, 5) == [2, 1, None]
    assert lg["plane"] == {(3, 1): b"AAA", (4, 3): b"BBB", (3, 2): b"DDD"} and lg["held"][3] == 0b111


def test_refusals_without_a_device():
    from summerset_b200 import _lib
    lib = _lib.load()

    def refused(rc, why):
        assert rc == _lib.SS_ERR_INVALID_ARG and why in lib.ss_last_error().decode(), (rc, lib.ss_last_error(), why)

    b = [16] * 4
    refused(lib.ss_engine_craft_recon_view_get(None, None), "null view")
    refused(lib.ss_engine_craft_recon_view_get(None, C.byref(_lib.CraftReconView())), "null engine")
    refused(lib.ss_engine_craft_step_up(None, None, 16, 1, 16, 32, 64, 16, None, 16), "null follower")
    refused(lib.ss_engine_craft_step_up(None, 16, 16, 1, 16, 32, 48, 16, None, 16), "multiple of 32")
    refused(lib.ss_engine_craft_step_up(None, 16, 16, 1, 16, 40, 64, 16, None, 16), "16-byte aligned")
    refused(lib.ss_engine_craft_step_up(None, 16, 16, 1, 16, 32, 64, 16, None, 16), "null engine")
    refused(lib.ss_engine_craft_reconstruct_reads(None, None, 0, 0, 4, 16, 0, *b, 1, None), "chunk_size")
    refused(lib.ss_engine_craft_reconstruct_reads(None, None, 0, 1, 1 << 16, 16, 0, *b, 1, None), "2^16")
    refused(lib.ss_engine_craft_reconstruct_reads(None, None, 0, 1, 4, 16, 0, *b, 1, None), "null engine")
    refused(lib.ss_follower_reconstruct_serve(None, 16, 0, 16, 16, 16, 1, 4, 5, 16, 0, 16, 16, 16, None), "null follower")
    refused(lib.ss_engine_craft_absorb(None, 16, 0, 16, 16, 16, 1, 1 << 16, 16, 16), "2^16")
    refused(lib.ss_engine_craft_absorb(None, 16, 0, 16, 16, 16, 1, 5, 16, 16), "null engine")


def test_no_device_without_a_context():
    from summerset_b200 import _lib
    lib = _lib.load()
    h = C.c_void_p()
    cfg = _lib.FollowerConfig(_lib.SS_PROTO_CRAFT, 5, 1, 0, 0, 1, 0, 1)
    rc = lib.ss_follower_create(None, C.byref(cfg), 4, C.byref(h))
    import torch
    assert rc == (_lib.SS_ERR_INVALID_ARG if torch.cuda.is_available() else _lib.SS_ERR_NO_DEVICE)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _ctx():
    from summerset_b200.api import Context
    return Context(0)


def _t(a, dt):
    import torch
    return torch.tensor(a, dtype=dt, device="cuda:0")


def _buf(frames, rng):
    """frames at odd offsets in one device buffer -> (buf, offsets)"""
    import torch
    buf, offs = bytearray(), []
    for x in frames:
        buf += bytes(rng.randint(0, 3))
        offs.append(len(buf))
        buf += x
    return _t(np.frombuffer(bytes(buf) + b"\0", dtype=np.uint8), torch.uint8), offs


@pytest.mark.gpu
def test_refusals_on_engines():
    import torch
    from summerset_b200 import _lib
    from summerset_b200.engine import Follower, LeaderEngine, RaftEngine
    ctx = _ctx()
    dev = "cuda:0"
    out = torch.zeros(4096, dtype=torch.uint8, device=dev)
    store = torch.zeros((5, 4096), dtype=torch.uint8, device=dev)
    fol = Follower(ctx, 4, 5, 1)
    g1, t1 = _t([0], torch.int32), _t([3], torch.int64)
    one = torch.zeros(1, dtype=torch.int64, device=dev)
    for e in (LeaderEngine(ctx, "rspaxos", 4, 5, 1, 16), RaftEngine(ctx, 4, 5, craft=False)):
        for call in (lambda: RaftEngine.recon_view(e), lambda: RaftEngine.step_up(e, fol, g1, t1, store),
                     lambda: RaftEngine.reconstruct_reads(e, out, 8, 1), lambda: RaftEngine.absorb(e, out, one, g1, g1.to(torch.uint8))):
            with pytest.raises(_lib.SummersetError, match="CRaft"):
                call()
        e.close()
    appended = RaftEngine(ctx, 4, 5, craft=True)
    appended.append(torch.ones(4, dtype=torch.int32, device=dev))
    for call in (lambda: appended.recon_view(), lambda: appended.step_up(fol, g1, t1, store),
                 lambda: appended.reconstruct_reads(out, 8, 1), lambda: appended.absorb(out, one, g1, g1.to(torch.uint8))):
        with pytest.raises(_lib.SummersetError, match="raft_append"):
            call()
    eng = RaftEngine(ctx, 4, 5, craft=True)
    for other, why in ((Follower(ctx, 4, 7, 1), "population"), (Follower(ctx, 8, 5, 1), "n_groups")):
        with pytest.raises(_lib.SummersetError, match=why):
            eng.step_up(other, g1, t1, store)
        other.close()
    with pytest.raises(_lib.SummersetError, match="multiple of 32"):
        eng.step_up(fol, g1, t1, torch.zeros((5, 4100), dtype=torch.uint8, device=dev))
    with pytest.raises(_lib.SummersetError, match="16-byte"):
        fol.reconstruct_serve(out, one, g1, g1.to(torch.uint8), out[1:])
    torch.cuda.synchronize()
    for e in (appended, eng, fol):
        e.close()


def _fol_state(fol):
    """the follower's state through its views -> [dict(start, le, ct, lc, ls, last_exec, term, dl, held, addr)]"""
    W = fol.W
    st, le, ct, lc, ls, lx = (x.cpu().tolist() for x in (fol.start_slot, fol.log_end, fol.curr_term, fol.last_commit, fol.last_snap,
                                                         fol.last_exec))
    term, dl, held, addr = (x.cpu().numpy() for x in (fol.term, fol.data_len, fol.held, fol.shard_addr))
    out = []
    for g in range(fol.G):
        rng_ = range(st[g], le[g]) if le[g] - st[g] <= W else range(0)
        pos = lambda s: s & (W - 1)
        out.append(dict(start=st[g], le=le[g], ct=ct[g], lc=lc[g], ls=ls[g], last_exec=lx[g],
                        term={s: int(term[g][pos(s)]) & ((1 << 64) - 1) for s in rng_}, dl={s: int(dl[g][pos(s)]) for s in rng_},
                        held={s: int(held[g][pos(s)]) & 0xFFFFFFFF for s in rng_}, addr={s: int(addr[g][pos(s)]) for s in rng_}))
    return out


def _check_step_up(eng, rv, lv, fols, listing, terms, o, store, stride, read_shard, before):
    """every engine word, ring entry and plane byte of a step-up against the restatement; groups not stepped up keep
    `before`"""
    G, W, T = eng.G, eng.W, eng.P + 1
    d = T // 2 + 1
    v, off, need, slots = step_up(fols, listing, terms, W, d, stride, G)
    assert o["verdict"].cpu().tolist() == v
    assert o["shard_off"].cpu().tolist() == [-1 if x is None else x for x in off] and int(o["need"][0]) == need
    now = _engine_words(eng, rv, lv)
    planes = store.cpu().numpy()
    base = store.data_ptr()
    done = {g: terms[i] for i, g in enumerate(listing) if v[i] == DONE}
    for g in range(G):
        if g not in done:
            assert all(np.array_equal(now[k][..., g] if k in ("next_slot", "try_next", "match") else now[k][g],
                                      before[k][..., g] if k in ("next_slot", "try_next", "match") else before[k][g]) for k in now), g
            continue
        fg = fols[g]
        assert (now["log_start"][g], now["log_end"][g], now["last_commit"][g], now["last_snap"][g], now["last_exec"][g],
                now["curr_term"][g]) == (fg["start"], fg["le"], fg["lc"], fg["ls"], fg["last_exec"], done[g])
        assert (now["next_slot"][:, g] == fg["le"]).all() and (now["try_next"][:, g] == fg["le"]).all() and (now["match"][:, g] == 0).all()
        assert now["last_recon"][g] == before["last_recon"][g]
        for s in range(fg["start"], fg["le"]):
            p_ = s & (W - 1)
            assert (now["terms"][g][p_], now["data_len"][g][p_], now["held"][g][p_], now["log_offset"][g][p_]) == \
                   (fg["term"][s], fg["dl"][s], fg["held"][s], 0), (g, s)
            if not fg["dl"][s]:
                assert now["shard_addr"][g][p_] == 0
                continue
            assert now["shard_addr"][g][p_] == base + slots[g][s]
            L = -(-fg["dl"][s] // d)
            for j in range(T):
                if fg["held"][s] >> j & 1:
                    got = planes[j][slots[g][s]:slots[g][s] + r16(L)].tobytes()
                    assert got[:L] == read_shard(g, s, j) and not any(got[L:]), (g, s, j)
    return v, slots


def _engine_words(eng, rv, lv):
    c = lambda x: x.cpu().numpy().copy()
    return dict(log_start=c(lv["log_start"]), log_end=c(eng.log_end), last_commit=c(eng.last_commit), last_snap=c(eng.last_snap),
                last_exec=c(eng.exec_view()["last_exec"]), curr_term=c(eng.curr_term), next_slot=c(eng.next_slot),
                try_next=c(lv["try_next"]), match=c(eng.match), last_recon=c(rv["last_recon"]), terms=c(eng.terms),
                data_len=c(lv["data_len"]), held=c(rv["held"]), shard_addr=c(lv["shard_addr"]), log_offset=c(lv["log_offset"]))


def _install(fol, groups, rng):
    """follower state through its views: groups[g] = dict(start, le, ct, lc, ls, last_exec, ent={slot: (term, batch,
    held)}); shards from the oracle's encoder in the store layout -> (store, {(g, s, j): shard bytes})"""
    import torch
    d, T, W = fol.d, fol.T, fol.W
    blob, addr, shards = bytearray(), {}, {}
    for g, gr in enumerate(groups):
        for s, (t, b, h) in gr["ent"].items():
            if not b:
                continue
            sh = tl.encode(b, d, T - d)
            L = len(sh[0])
            blob += bytes(rng.choice((0, 16, 32)))
            addr[(g, s)] = len(blob)
            for j in range(T):
                shards[(g, s, j)] = sh[j]
                if h >> j & 1:
                    blob += sh[j] + bytes(pitch(L) - L)
    store = torch.tensor(np.frombuffer(bytes(blob) + bytes(64), dtype=np.uint8), device="cuda:0")
    base = store.data_ptr()
    G = len(groups)
    arr = {k: np.zeros((G, W), dtype=np.int64) for k in ("term", "shard_addr")}
    arr.update({k: np.zeros((G, W), dtype=np.int32) for k in ("held", "data_len")})
    for g, gr in enumerate(groups):
        for s, (t, b, h) in gr["ent"].items():
            p_ = s & (W - 1)
            arr["term"][g][p_] = np.int64(np.uint64(t))
            arr["held"][g][p_], arr["data_len"][g][p_] = np.int32(np.uint32(h)), len(b)
            arr["shard_addr"][g][p_] = base + addr.get((g, s), 0) if b else 0
    for k, a in arr.items():
        getattr(fol, k).copy_(torch.tensor(a, device="cuda:0"))
    for k in ("start", "le", "ct", "lc", "ls", "last_exec"):
        dst = dict(start=fol.start_slot, le=fol.log_end, ct=fol.curr_term, lc=fol.last_commit, ls=fol.last_snap, last_exec=fol.last_exec)[k]
        dst.copy_(torch.tensor(np.array([gr[k] for gr in groups], dtype=np.uint64).view(np.int64), device="cuda:0"))
    return store, shards


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 5, 7, 9, 12])
def test_step_up_matches_the_restatement(n):
    import torch
    from summerset_b200.engine import Follower, RaftEngine
    ctx = _ctx()
    d, T = n // 2 + 1, n
    rng = random.Random(500 + n)
    G, W, FW = 24, 16, 32
    fol = Follower(ctx, G, n, 1, window=FW)
    groups = []
    for g in range(G):
        start = rng.choice((0, 3, 30, 1000))                      # logs that wrap both rings
        span = rng.choice((1, 2, 5, W - 1, W)) if g != 1 else W + 1
        ent = {}
        t = 1
        for s in range(start, start + span):
            t += rng.random() < 0.3
            b = b"" if s == 0 or rng.random() < 0.08 else rng.randbytes(rng.choice((1, 17, 100, 4096)))
            h = rng.choice((0, 1 << rng.randrange(T), (1 << d) - 1, (1 << T) - 1, rng.randrange(1 << T)))
            ent[s] = (t, b, h if b else 0)
        le = start + span
        groups.append(dict(start=start, le=le, ct=t + rng.choice((0, 1)), lc=max(start, le - 1 - rng.randint(0, 2)), ls=start,
                           last_exec=start, ent=ent))
    groups[2]["ent"][groups[2]["start"]] = (1 << 32, b"x", 1)      # a term past the engine's u32 ring
    groups[3]["ct"] = 1 << 40                                     # above every term the listing offers
    store_f, shards = _install(fol, groups, rng)
    fols = _fol_state(fol)
    eng = RaftEngine(ctx, G, n, craft=True, window=W)
    rv, lv = eng.recon_view(), eng.log_view()
    rv["last_recon"].copy_(torch.arange(G, dtype=torch.int64, device="cuda:0"))
    listing = list(range(G)) + [5, G, G + 7, 0]                   # repeats and groups past n_groups
    rng.shuffle(listing)
    terms = [5 if g == 3 else max(fols[g]["ct"], 1) if g < G else 5 for g in listing]
    need = sum(pitch(-(-fg["dl"][s] // d)) for fg in fols for s in fg["dl"] if fg["dl"][s])
    for stride in ((need + 64) // 32 * 32 + 32, max(32, need // 2 // 32 * 32)):
        before = _engine_words(eng, rv, lv)
        store = torch.zeros((T, stride), dtype=torch.uint8, device="cuda:0")
        ctx.device_status()
        o = eng.step_up(fol, _t(listing, torch.int32), _t(terms, torch.int64), store)
        torch.cuda.synchronize()
        v, _ = _check_step_up(eng, rv, lv, fols, listing, terms, o, store, stride, lambda g, s, j: shards[(g, s, j)], before)
        assert {WINDOW, RANGE, STALE, IGNORED, DONE} <= set(v)
        assert (STORE_FULL in v) == bool(ctx.device_status() & STATUS_STORE_FULL)
        eng.close()
        eng = RaftEngine(ctx, G, n, craft=True, window=W)
        rv, lv = eng.recon_view(), eng.log_view()
    assert _fol_state(fol) == fols                                 # the follower's state is only read
    del store_f
    eng.close()
    fol.close()


def _serve_absorb_case(n, seed):
    """a stepped-up leader and a follower that holds other shards of the same entries"""
    import torch
    from summerset_b200.engine import Follower, RaftEngine
    ctx = _ctx()
    d, T = n // 2 + 1, n
    rng = random.Random(seed)
    G, W = 12, 32
    src, peer = Follower(ctx, G, n, 1, window=W), Follower(ctx, G, n, 2, window=W)
    base, pgroups = [], []
    for g in range(G):
        start = rng.choice((1, 20, 40))
        ent, pent = {}, {}
        for s in range(start, start + rng.randint(3, 12)):
            b = rng.randbytes(rng.choice((1, 31, 500, 3000)))
            t = 1 + (s - start) // 4
            ent[s] = (t, b, 1 << rng.randrange(T))
            pent[s] = (t + (rng.random() < 0.1), b, rng.randrange(1, 1 << T))   # a few entries of another term
        le = max(ent) + 1
        base.append(dict(start=start, le=le, ct=t, lc=le - 1, ls=start, last_exec=start - 1, ent=ent))
        pgroups.append(dict(start=start, le=le, ct=t, lc=start - 1, ls=start, last_exec=start - 1, ent=pent))
    st1, shards = _install(src, base, rng)
    st2, _ = _install(peer, pgroups, rng)
    eng = RaftEngine(ctx, G, n, craft=True, window=W)
    stride = 1 << 20
    store = torch.zeros((T, stride), dtype=torch.uint8, device="cuda:0")
    o = eng.step_up(src, _t(list(range(G)), torch.int32), _t([9] * G, torch.int64), store)
    torch.cuda.synchronize()
    assert o["verdict"].cpu().tolist() == [DONE] * G
    return ctx, eng, src, peer, store, shards, _fol_state(src), _fol_state(peer), [st1, st2], rng


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5, 7])
def test_serve_and_absorb_match_the_restatement(n):
    import torch
    ctx, eng, src, peer, store, shards, fs, fp, keep, rng = _serve_absorb_case(n, 800 + n)
    G, W, d, T = eng.G, eng.W, n // 2 + 1, n
    rv, lv = eng.recon_view(), eng.log_view()
    # recon reads: every committed entry holding fewer than d shards, in two calls (chunk 3), the second with nothing new
    lgs = [dict(last_exec=f["last_exec"], start=f["start"], last_recon=0, lc=f["lc"], held=dict(f["held"]), term=f["term"]) for f in fs]
    out = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda:0")
    listed = [recon_walk(lg, d) for lg in lgs]
    r = eng.reconstruct_reads(out, 256, 3, groups=_t([3, 1, G + 2, 3] + [g for g in range(G) if g not in (1, 3)], torch.int32))
    torch.cuda.synchronize()
    order = [3, 1, 3] + [g for g in range(G) if g not in (1, 3)]   # group 3 listed twice: planned twice from the same state
    want = [(g, x) for g in order for x in recon_frames(listed[g], 3)]
    assert int(r["totals"][0]) == len(want)
    on = out.cpu().numpy()
    for k, (g, x) in enumerate(want):
        off = int(r["frame_off"][k])
        assert (int(r["frame_group"][k]), int(r["frame_dst"][k]), int(r["frame_len"][k])) == (g, 0xFF, len(x))
        assert on[off:off + len(x)].tobytes() == x
    assert rv["last_recon"].cpu().tolist() == [lg["last_recon"] for lg in lgs]
    assert int(eng.reconstruct_reads(out, 256, 3)["totals"][0]) == 0
    # the capacity cut: a suffix of the groups writes nothing and keeps last_recon
    rv["last_recon"].zero_()
    ctx.device_status()
    r = eng.reconstruct_reads(out, 256, 3, out_capacity=200)
    torch.cuda.synchronize()
    assert ctx.device_status() & STATUS_FRAME_OVERFLOW
    lr, nf = rv["last_recon"].cpu().tolist(), int(r["totals"][0])
    fo, fgr, fl = (r[k][:nf].cpu().tolist() for k in ("frame_off", "frame_group", "frame_len"))
    written = {g for g, o_ in zip(fgr, fo) if o_ != -1}
    cut = {g for g, o_ in zip(fgr, fo) if o_ == -1}
    assert written and cut and not written & cut and max(written) < min(cut)
    assert all(o_ + r16(x) <= 200 for o_, x in zip(fo, fl) if o_ != -1) and all(x == 0 for o_, x in zip(fo, fl) if o_ == -1)
    assert all(lr[g] == (lgs[g]["last_recon"] if g in written else 0) for g in range(G))
    # serve: shuffled requests over every group with out-of-log slots, other terms and repeats
    reqs = []
    for g in range(G):
        f = fp[g]
        sl = [(s, f["term"][s]) for s in range(f["start"], f["le"])]
        sl += [(f["start"] - 1, 1), (f["le"], 1), (f["start"], f["term"][f["start"]] + 1)] + rng.sample(sl, 2)
        rng.shuffle(sl)
        reqs += [(g, sl[:k]) for k in (len(sl), 3)]
    rng.shuffle(reqs)
    frames = [reconstruct(x) for _, x in reqs] + [reconstruct([(1, 1)], variant=7), framed(vi(2)), framed(reconstruct([(1, 1)])[8:-1])]
    grp = [g for g, _ in reqs] + [0, 0, 0]
    buf, offs = _buf(frames, rng)
    rout = torch.full((1 << 20,), 0xA5, dtype=torch.uint8, device="cuda:0")
    s_ = peer.reconstruct_serve(buf, _t(offs, torch.int64), _t(grp, torch.int32), _t([0] * len(grp), torch.uint8), rout)
    torch.cuda.synchronize()
    ro = rout.cpu().numpy()
    pstore, pbase = keep[1].cpu().numpy(), keep[1].data_ptr()

    def pshard(g, s, j):                                          # the peer's shard j, by rank in its store slot
        L = -(-fp[g]["dl"][s] // d)
        at = fp[g]["addr"][s] - pbase + popc(fp[g]["held"][s] & ((1 << j) - 1)) * pitch(L)
        return pstore[at:at + L].tobytes()

    replies = []
    for i, (g, sl) in enumerate(reqs):
        want = serve(fp[g], sl, d, T, lambda s, j: pshard(g, s, j))
        assert int(s_["verdict"][i]) & 0xFFFFFFFF == ACCEPTED
        if want is None:
            assert int(s_["reply_len"][i]) == 0 and int(s_["reply_off"][i]) == -1
            continue
        off = int(s_["reply_off"][i])
        assert int(s_["reply_len"][i]) == len(want) and ro[off:off + len(want)].tobytes() == want, i
        replies.append((g, want))
    v = [int(x) & 0xFFFFFFFF for x in s_["verdict"][len(reqs):].cpu().tolist()]
    assert v == [7, 0x80000002, MALFORMED]
    # the out_capacity cut: the replies whose regions end past it are a suffix, not written, OUT_FULL
    offs_all, lens_all = s_["reply_off"].cpu().tolist(), s_["reply_len"].cpu().tolist()
    with_reply = [i for i in range(len(reqs)) if lens_all[i]]
    cap = offs_all[with_reply[len(with_reply) // 2]]
    ctx.device_status()
    c_ = peer.reconstruct_serve(buf, _t(offs, torch.int64), _t(grp, torch.int32), _t([0] * len(grp), torch.uint8), rout, out_capacity=cap)
    torch.cuda.synchronize()
    assert ctx.device_status() & STATUS_FRAME_OVERFLOW
    for i in with_reply:
        kept = offs_all[i] + r16(lens_all[i]) <= cap
        assert (int(c_["verdict"][i]) & 0xFFFFFFFF, int(c_["reply_off"][i]), int(c_["reply_len"][i])) == \
               ((ACCEPTED, offs_all[i], lens_all[i]) if kept else (OUT_FULL, -1, 0)), i
    assert int(c_["total"][0]) == int(s_["total"][0])
    # absorb: the replies in shuffled order, with malformed ones of every kind and duplicate carriers
    bad = _bad_replies(d, T)
    assert all(parse_reply(x, d, T) is None for x in bad)
    pool = [(g, x) for g, x in replies] + [(rng.randrange(G), x) for x in bad] + [(G + 1, replies[0][1])]
    pool += [(g, x) for g, x in rng.sample(replies, 3)]
    rng.shuffle(pool)
    # first carriers whose shard lengths are spelled as non-minimal varints (3, 5 and 9 bytes), which decode as well
    for g in (0, 1):
        s0 = fs[g]["start"]
        L = -(-fs[g]["dl"][s0] // d)
        missing = [j for j in range(T) if not fs[g]["held"][s0] >> j & 1]
        sh = {j: rng.randbytes(L) for j in missing[:3]}
        pool.insert(0, (g, reconstruct_reply([(s0, codeword_wide(d, T - d, fs[g]["dl"][s0], sh, (251, 252, 253)))])))
    lgs = [dict(start=fs[g]["start"], le=fs[g]["le"], dl=dict(fs[g]["dl"]), held=dict(fs[g]["held"]), plane={}) for g in range(G)]
    want_abs = [None] * len(pool)
    for g in range(G):
        idx = [i for i, (h, _) in enumerate(pool) if h == g]
        for i, a in zip(idx, absorb(lgs[g], [pool[i][1] for i in idx], d, T)):
            want_abs[i] = a
    buf, offs = _buf([x for _, x in pool], rng)
    a = eng.absorb(buf, _t(offs, torch.int64), _t([g for g, _ in pool], torch.int32), _t([1] * len(pool), torch.uint8))
    torch.cuda.synchronize()
    for i, w in enumerate(want_abs):
        ver = int(a["verdict"][i]) & 0xFFFFFFFF
        if w is None:
            assert ver != ACCEPTED and int(a["absorbed"][i]) == 0, i
        else:
            assert ver == ACCEPTED and int(a["absorbed"][i]) == w, i
    held, addr = rv["held"].cpu().numpy(), lv["shard_addr"].cpu().numpy()
    planes, sbase = store.cpu().numpy(), store.data_ptr()
    for g in range(G):
        for s in range(lgs[g]["start"], lgs[g]["le"]):
            assert int(held[g][s & (W - 1)]) & 0xFFFFFFFF == lgs[g]["held"][s], (g, s)
            for (s2, j), x in lgs[g]["plane"].items():
                if s2 == s:
                    o_ = int(addr[g][s & (W - 1)]) - sbase
                    got = planes[j][o_:o_ + r16(len(x))].tobytes()
                    assert got[:len(x)] == x and not any(got[len(x):])
    for o in (eng, src, peer):
        o.close()
    del keep


def _bad_replies(d, T):
    """ReconstructReply frames that absorb nothing, each malformed in one way (or another message)"""
    L = 4
    ok = tf.codeword(d, T - d, 4 * d, {0: b"\x01" * L})              # d, p, data_len, L, T: one byte each; shard 0's tag at 5
    body = lambda cw: vi(0) + vi(5) + vi(1) + vi(5) + cw
    good = lambda cw: framed(body(cw))
    return [framed(body(ok)[:-1]),                                # truncated
            framed(body(ok) + b"\x00"),                            # a trailing byte
            good(bytes([d + 1]) + ok[1:]),                        # another code
            good(ok[:3] + vi(L + 1) + ok[4:]),                    # shard_len != ceil(data_len / d)
            good(ok[:4] + vi(T - 1) + ok[5:]),                    # T - 1 shard Options
            good(ok[:5] + b"\x02" + ok[6:]),                      # an Option tag other than 0 / 1
            good(ok[:6] + vi(L - 1) + ok[7:7 + L - 1] + ok[7 + L:]),   # a present shard of another length
            good(ok[:-1] + b"\x02"),                              # a data_copy tag other than 0 / 1
            good(with_data_copy(ok, b"\x00" * (4 * d - 1))),      # data_copy Some, one byte short
            framed(vi(0) + vi(5) + vi(2) + vi(5) + ok),           # two entries announced, one sent
            reconstruct_reply([(5, ok)], variant=6),              # another PeerMsg
            framed(vi(1) + vi(0))]                                # another PeerMessage


def _failover(n, full_copy):
    """A device leader replicates several terms of entries to device followers, frames to one follower dropped so the
    logs diverge; the leader is discarded, the Raft vote rule picks the winner from the follower views, and the winner's
    engine steps up, commits one entry of its term, reads back the shards it lacks and executes every batch."""
    import torch
    from summerset_b200.engine import Follower, RaftEngine, append_reply_parse
    ctx = _ctx()
    G, W, chunk = 16, 64, 4
    d, T = n // 2 + 1, n
    rng = random.Random(4000 + 10 * n + full_copy)
    dev = "cuda:0"
    fols = {r: Follower(ctx, G, n, r, window=W) for r in range(1, n)}
    keep, batch = [], {}
    stride = G * pitch(-(-3000 // d)) * 8                       # every plane call of a log takes the same stride

    def propose(eng, me, fc=full_copy):
        lens = [rng.choice((1, 15, 16, 17, 300, 3000)) for _ in range(G)]
        store, got = _propose(eng, me, lens, stride, fc)
        keep.append(store)
        for g, (s, b) in got.items():
            batch[(g, s)] = b

    def round_trip(eng, me, live, want=None, heartbeat=False, fc=full_copy):
        """pack, deliver to the live replicas, ingest the replies, back off -> (want_end or None, frames to each replica)"""
        out = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
        o = eng.pack_append(me, out, 1 << 12, want_end=want, heartbeat=heartbeat, full_copy=fc, msg_chunk_size=chunk)
        torch.cuda.synchronize()
        nf = int(o["n_frames"][0])
        fo, fg, fp = o["frame_off"][:nf], o["frame_group"][:nf], o["frame_peer"][:nf]
        on, sent, replies = out.cpu().numpy(), {}, []
        for r in live:
            q = r if r < me else r - 1
            sel = (fp == q).nonzero().flatten()
            sent[r] = [(int(fg[i]), on[int(fo[i]):int(fo[i]) + int(o["frame_len"][i])].tobytes()) for i in sel.tolist()]
            if sel.numel() == 0:
                continue
            st, wal = torch.zeros(1 << 22, dtype=torch.uint8, device=dev), torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
            keep.append(st)
            a = fols[r].append(out, fo[sel].contiguous(), fg[sel].contiguous(), torch.full_like(fp[sel], me), st, wal)
            torch.cuda.synchronize()
            rl, cells = a["reply_len"].cpu().numpy(), a["replies"].cpu().numpy()
            for i, g in enumerate(fg[sel].cpu().tolist()):
                replies.append((g, q, cells[i][:rl[i]].tobytes()))
        if not replies:
            return None, sent
        tb, offs = _buf([x for _, _, x in replies], rng)
        fo2, fg2, fp2 = _t(offs, torch.int64), _t([r[0] for r in replies], torch.int32), _t([r[1] for r in replies], torch.uint8)
        rec = append_reply_parse(ctx, tb, fo2, fg2, fp2, eng.curr_term, G)
        eng.on_append_replies(rec["rec_group"], rec["rec_peer"], rec["rec_end_slot"])
        want = eng.backoff(tb, fo2, fg2, fp2, rec["rec_kind"])
        eng.tick()
        torch.cuda.synchronize()
        return (want if (want != -1).any() else None), sent

    def settle(eng, me, live, fc=full_copy):
        want, _ = round_trip(eng, me, live, fc=fc)
        for _ in range(8):
            if want is None:
                break
            want, _ = round_trip(eng, me, live, want, fc=fc)
        assert want is None
        round_trip(eng, me, live, heartbeat=True, fc=fc)

    # 1. the first leader, replica 0: three terms of entries; replica 1 misses the first term's second round (it catches
    #    up through a back-off), replica n - 1 misses the whole last term.  The code survives n - d lost shards: from
    #    n = 5 up, the crashed leader's and the lagging replica's.  At n = 3 and 4 coded copies of the last term would not
    #    survive both, so that term goes out in full copy, CRaft's fallback: the new leader holds its d data shards
    old = RaftEngine(ctx, G, n, craft=True, window=W)
    old.log_view()
    lag = n - 1
    for term in (1, 2, 3):
        fc = full_copy or (term == 3 and n - d < 2)
        old.set_full_copy(fc)
        old.curr_term.fill_(term)
        for k in range(2):
            propose(old, 0, fc)
            live = [r for r in fols if not (term == 1 and k == 1 and r == 1) and not (term == 3 and r == lag)]
            settle(old, 0, live, fc)
    old.close()
    # 2. the vote rule over the survivors' logs: the highest (last term, last slot), the lowest id among equals
    views = {r: _fol_state(f) for r, f in fols.items()}
    key = lambda r, g: (views[r][g]["term"][views[r][g]["le"] - 1], views[r][g]["le"] - 1)
    winners = {max(fols, key=lambda r: (key(r, g), -r)) for g in range(G)}
    assert len(winners) == 1
    w = winners.pop()
    assert w != lag and all(key(lag, g) < key(w, g) for g in range(G))
    new_term = max(max(v[g]["ct"] for g in range(G)) for v in views.values()) + 1
    eng = RaftEngine(ctx, G, n, craft=True, window=W)
    rv, lv = eng.recon_view(), eng.log_view()
    before = _engine_words(eng, rv, lv)
    planes = torch.zeros((T, stride), dtype=torch.uint8, device=dev)
    listing = list(range(G))
    o = eng.step_up(fols[w], _t(listing, torch.int32), _t([new_term] * G, torch.int64), planes)
    torch.cuda.synchronize()
    coded = _Coded(batch, d, T)
    v, _ = _check_step_up(eng, rv, lv, views[w], listing, [new_term] * G, o, planes, stride,
                          lambda g, s, j: coded[(g, s)][j], before)
    assert v == [DONE] * G
    if full_copy:
        eng.set_full_copy(True)
    # 3. one entry in the new term; the lagging follower's back-off resend carries only the shards the new leader holds
    survivors = [r for r in fols if r != w]
    propose(eng, w)
    want, _ = round_trip(eng, w, survivors)
    ql = lag if lag < w else lag - 1
    assert want is not None and int(want[ql].max()) >= 0
    st = dict(terms=eng.terms.cpu().numpy(), held=rv["held"].cpu().numpy(), dl=lv["data_len"].cpu().numpy(),
              lc=eng.last_commit.cpu().tolist(), ls=eng.last_snap.cpu().tolist(), ns=eng.next_slot.cpu().numpy(),
              tn=lv["try_next"].cpu().numpy(), le=eng.log_end.cpu().tolist(), ct=eng.curr_term.cpu().tolist())
    want_np = want.cpu().numpy()
    _, sent = round_trip(eng, w, survivors, want)
    wanted = (1 << d) - 1 if full_copy else 1 << lag
    frames = []
    for g in range(G):
        t = max(int(st["tn"][ql][g]), int(st["ns"][ql][g]))
        end = min(int(want_np[ql][g]), st["le"][g] - 1)
        for first in range(t, end + 1, chunk):
            ents = []
            for s in range(first, min(end, first + chunk - 1) + 1):
                p_ = s & (W - 1)
                held = int(st["held"][g][p_]) & wanted
                ents.append(tf.entry(int(st["terms"][g][p_]), d, T - d, int(st["dl"][g][p_]),
                                     {j: coded[(g, s)][j] for j in range(T) if held >> j & 1}, False, 0))
            prev = first - 1
            frames.append((g, tf.append_entries(st["ct"][g], prev, int(st["terms"][g][prev & (W - 1)]), ents, st["lc"][g], st["ls"][g])))
    assert sent[lag] == frames and frames
    if not full_copy:                                             # old entries go out without the lagging replica's shard
        assert any(b"\x00" * 2 in x for _, x in frames)
    settle(eng, w, survivors)
    le = eng.log_end.cpu().tolist()
    assert eng.last_commit.cpu().tolist() == [x - 1 for x in le]
    # 4. reconstruct reads to the survivors, their replies absorbed, then every batch executes
    out = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
    r = eng.reconstruct_reads(out, 1 << 12, chunk)
    torch.cuda.synchronize()
    nf = int(r["totals"][0])
    assert (nf == 0) == full_copy
    if nf:
        fo, fg = r["frame_off"][:nf], r["frame_group"][:nf]
        assert (r["frame_dst"][:nf] == 0xFF).all()
        replies = []
        for q_r in survivors:
            rout = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
            s_ = fols[q_r].reconstruct_serve(out, fo, fg, torch.full((nf,), w, dtype=torch.uint8, device=dev), rout)
            torch.cuda.synchronize()
            ro = rout.cpu().numpy()
            for i in range(nf):
                ln = int(s_["reply_len"][i])
                if ln:
                    off = int(s_["reply_off"][i])
                    replies.append((int(fg[i]), q_r if q_r < w else q_r - 1, ro[off:off + ln].tobytes()))
        rng.shuffle(replies)
        tb, offs = _buf([x for _, _, x in replies], rng)
        a = eng.absorb(tb, _t(offs, torch.int64), _t([x[0] for x in replies], torch.int32), _t([x[1] for x in replies], torch.uint8))
        torch.cuda.synchronize()
        assert (a["verdict"].cpu().numpy().view(np.uint32) == ACCEPTED).all() and int(a["absorbed"].sum()) > 0
    held = rv["held"].cpu().numpy()
    assert all(popc(int(held[g][s & (W - 1)])) >= d for g in range(G) for s in range(1, le[g]))
    res = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
    ex = eng.execute(res, 1 << 12)
    torch.cuda.synchronize()
    nrec = int(ex["totals"][0])
    assert nrec == len(batch) == sum(x - 1 for x in le)
    recs = list(zip(*(ex[k][:nrec].cpu().tolist() for k in ("rec_group", "rec_slot", "rec_off", "rec_len"))))
    assert [(g, s_) for g, s_, _, _ in recs] == sorted(batch)        # every group's batches, in slot order
    rn = res.cpu().numpy()
    for g, s_, off, dl in recs:
        assert rn[off:off + dl].tobytes() == batch[(g, s_)], (g, s_)
    assert eng.exec_view()["last_exec"].cpu().tolist() == [x - 1 for x in le]
    for f in fols.values():
        f.close()
    eng.close()


class _Coded(dict):
    """every shard of a batch, coded on first use"""

    def __init__(self, batch, d, T):
        super().__init__()
        self.batch, self.d, self.T = batch, d, T

    def __missing__(self, k):
        self[k] = tl.encode(self.batch[k], self.d, self.T - self.d)
        return self[k]


def _propose(eng, me, lens, stride, full_copy):
    import torch
    rng = random.Random(sum(lens))
    batches = [rng.randbytes(x) for x in lens]
    arena, offs = bytearray(), []
    for b in batches:
        offs.append(len(arena))
        arena += b
    store = torch.zeros((eng.P + 1, stride), dtype=torch.uint8, device="cuda:0")
    o = eng.propose(me, _t(np.frombuffer(bytes(arena), dtype=np.uint8), torch.uint8), _t(offs, torch.int64), _t(lens, torch.int32), store,
                    torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0"), full_copy=full_copy)
    slots = o["slot_out"].cpu().tolist()
    assert min(slots) >= 0
    return store, {g: (slots[g], batches[g]) for g in range(len(lens))}


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5, 7])
@pytest.mark.parametrize("full_copy", [False, True])
def test_closed_loop_fail_over(n, full_copy):
    _failover(n, full_copy)
