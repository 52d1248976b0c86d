"""WAL recovery on the CRaft follower (ss_follower_recover).

`recover_batch` restates recover_from_wal (craft/recovery.rs:11-165) per group over the follower's ring and the rules of
include/summerset_b200.h: the Metadata record first, LogEntry record k at slot start_slot + k, the log ending at the
first record that breaks this, the whole-group refusal past the window and the per-group store cut.  `parse_record`
restates the entry rules of ss_follower_append.  The record encoders are pinned to tests/test_follower.py's and to
hand-worked bytes.  GPU tests compare every state word and every shard byte read through shard_addr with the
restatement, inside canary bytes, and replay the WALs a live cluster wrote into fresh followers.
"""
from __future__ import annotations

import random

import numpy as np
import pytest

from summerset_b200 import _lib
from tests import test_follower as tf

vi, framed = tf.vi, tf.framed
ACC, BEYOND, STORE_FULL = tf.ACCEPTED, tf.BEYOND, tf.STORE_FULL
MALFORMED = tf.MALFORMED
AFTER_END = _lib.SS_RECOVER_VERDICT_AFTER_END
ST_STORE_FULL, ST_OVERFLOW = 16, 4                 # SS_DEV_STATUS_STORE_FULL, SS_DEV_STATUS_FRAME_OVERFLOW
NONE = 0xFF
MAX_BODY = (1 << 32) - 1 - 64


def pitch(L):
    return (L + 31) & ~31


def r16(x):
    return (x + 15) & ~15


# ---- record encoders --------------------------------------------------------------------------------------------
def meta_record(curr_term, voted_for=NONE, variant=0) -> bytes:
    """DurEntry::Metadata{curr_term, voted_for} as the device's 32-byte cells hold it (without the zero tail)"""
    return framed(vi(variant) + vi(curr_term) + bytes([voted_for]))


def log_record(term, d, p, data_len, shards, external=False, log_offset=0, variant=1) -> bytes:
    """DurEntry::LogEntry{LogEntry{term, reqs_cw, external, log_offset}}"""
    return framed(vi(variant) + tf.entry(term, d, p, data_len, shards, external, log_offset))


def null_record(d, p, variant=1) -> bytes:
    """the slot-0 null entry an empty WAL gets (recovery.rs:99-125)"""
    return log_record(0, d, p, 0, {}, False, 0, variant)


def shards_of(rng, d, T, data_len, held):
    L = -(-data_len // d)
    return {j: rng.randbytes(L) for j in range(T) if (held >> j) & 1}


# ---- the parse and replay restatement ------------------------------------------------------------------------------
def _vget(b, n):
    if n >= len(b):
        return None
    t = b[n]
    if t < 251:
        return t, n + 1
    nb = {251: 2, 252: 4, 253: 8}.get(t)
    if nb is None or len(b) - n - 1 < nb:
        return None
    return int.from_bytes(b[n + 1:n + 1 + nb], "little"), n + 1 + nb


def parse_record(buf: bytes, off: int, d: int, T: int, mv: int, lv: int):
    """-> ("meta", curr_term, voted_for) | ("log", term, data_len, {j: shard}) | None for a malformed record"""
    if off > len(buf) or len(buf) - off < 8:
        return None
    ln = int.from_bytes(buf[off:off + 8], "big")
    if ln > len(buf) - off - 8 or ln > MAX_BODY:
        return None
    b = buf[off + 8:off + 8 + ln]
    r = _vget(b, 0)
    if r is None:
        return None
    v, n = r
    if v == mv:
        r = _vget(b, n)
        if r is None or len(b) - r[1] != 1:
            return None
        return ("meta", r[0], b[r[1]])
    if v != lv:
        return None
    r = _vget(b, n)
    if r is None:
        return None
    term, n = r
    if len(b) - n < 2 or b[n] != d or b[n + 1] != T - d:
        return None
    n += 2
    f = []
    for _ in range(3):
        r = _vget(b, n)
        if r is None:
            return None
        f.append(r[0])
        n = r[1]
    dl, sl, cnt = f
    if dl >= 1 << 32 or cnt != T or sl != -(-dl // d):
        return None
    shards = {}
    for j in range(T):
        if n >= len(b):
            return None
        tag = b[n]
        n += 1
        if tag == 0:
            continue
        if tag != 1:
            return None
        r = _vget(b, n)
        if r is None or r[0] != sl or len(b) - r[1] < sl:
            return None
        n = r[1]
        shards[j] = bytes(b[n:n + sl])
        n += sl
    if n >= len(b) or b[n] != 0:                                      # data_copy None
        return None
    n += 1
    if n >= len(b) or b[n] > 1:                                       # external
        return None
    n += 1
    r = _vget(b, n)                                                   # log_offset
    if r is None or r[1] != len(b):
        return None
    return ("log", term, dl, shards)


def recover_group(parsed, W):
    """one group's records (parsed) -> (verdicts, meta, entries); entries [] and verdicts BEYOND for a refused group"""
    verdicts, meta, ents, ended = [], None, [], False
    for k, r in enumerate(parsed):
        if ended:
            verdicts.append(AFTER_END)
        elif r is not None and r[0] == ("meta" if k == 0 else "log"):
            verdicts.append(ACC)
            if k == 0:
                meta = r
            else:
                ents.append(r)
        else:
            verdicts.append(MALFORMED)
            ended = True
    if len(ents) > W:
        return [BEYOND] * len(parsed), None, [], True
    return verdicts, meta, ents, False


def ent_bytes(e, d):
    return len(e[3]) * pitch(-(-e[2] // d))


def recover_batch(buf, offs, groups, G, W, d, T, mv, lv, cap):
    """-> verdicts, total, status, applied {g: (meta, entries, group offset)}"""
    by = {}
    for i, g in enumerate(groups):
        by.setdefault(g, []).append(i)
    verdicts, status, applied, region = [None] * len(groups), 0, {}, {}
    for g, idx in by.items():
        if g >= G:
            for i in idx:
                verdicts[i] = MALFORMED
            continue
        v, meta, ents, over = recover_group([parse_record(buf, offs[i], d, T, mv, lv) for i in idx], W)
        status |= ST_OVERFLOW if over else 0
        for i, x in zip(idx, v):
            verdicts[i] = x
        region[g] = (meta, ents, sum(ent_bytes(e, d) for e in ents))
    off = 0
    for g in sorted(region):
        meta, ents, nb = region[g]
        if off + nb > cap:
            for i in by[g]:
                if verdicts[i] == ACC:
                    verdicts[i] = STORE_FULL
                    status |= ST_STORE_FULL
        elif meta is not None:
            applied[g] = (meta, ents, off)
        off += nb
    return verdicts, off, status, applied


def test_record_bytes_pinned():
    assert meta_record(7) == tf.dur_metadata(7) and meta_record(300, NONE, 251) == tf.dur_metadata(300, 251)
    e = tf.Ent(5, 3, 2, 10, {0: bytes(4), 4: b"abcd"}, external=False)
    assert log_record(5, 3, 2, 10, e.shards) == tf.dur_log_entry(e.to_external())
    assert log_record(5, 3, 2, 10, e.shards, variant=65535) == tf.dur_log_entry(e.to_external(), 65535)
    # the 32-byte Metadata cell at curr_term 300, voted_for 2: length 5, variant 0, fb 2c 01, 02, zero to the end
    cell = meta_record(300, 2) + bytes(32 - 13)
    assert cell == bytes([0, 0, 0, 0, 0, 0, 0, 5, 0, 0xFB, 0x2C, 0x01, 2]) + bytes(19)
    assert meta_record(1 << 32, 0, 65535) == bytes([0] * 7 + [13, 0xFB, 0xFF, 0xFF, 0xFD, 0, 0, 0, 0, 1, 0, 0, 0, 0])
    assert null_record(2, 1) == framed(bytes([1, 0, 2, 1, 0, 0, 3, 0, 0, 0, 0, 0, 0]))


def test_parse_record_rules():
    d, T = 3, 5
    good = log_record(4, d, T - d, 10, {1: b"abcd"})
    assert parse_record(good, 0, d, T, 0, 1) == ("log", 4, 10, {1: b"abcd"})
    assert parse_record(meta_record(9, 4), 0, d, T, 0, 1) == ("meta", 9, 4)
    assert parse_record(good[:-1], 0, d, T, 0, 1) is None                            # partial
    assert parse_record(framed(good[8:] + b"\0"), 0, d, T, 0, 1) is None             # trailing bytes
    assert parse_record(good, 0, d, T, 0, 2) is None                                 # foreign variant
    assert parse_record(good, 0, 2, T, 0, 1) is None                                 # another code
    assert parse_record(framed(good[8:-2] + b"\x02\x00"), 0, d, T, 0, 1) is None     # external 2
    nm = framed(b"\xfb\x01\x00" + good[9:])                                          # non-minimal variant
    assert parse_record(nm, 0, d, T, 0, 1) == ("log", 4, 10, {1: b"abcd"})


def test_model_rules():
    d, T, W = 2, 3, 2
    m, e = meta_record(3, 1), log_record(3, d, T - d, 3, {0: b"ab"})
    buf = m + e + e + m + e
    offs = [0, len(m), len(m) + len(e), len(m) + 2 * len(e), 2 * len(m) + 2 * len(e)]
    v, total, st, ap = recover_batch(buf, offs, [0, 0, 0, 0, 0], 1, W, d, T, 0, 1, 1 << 30)
    assert v == [ACC, ACC, ACC, MALFORMED, AFTER_END] and total == 2 * pitch(2) and st == 0
    v, total, st, ap = recover_batch(buf, offs[:3] + offs[4:], [0, 0, 0, 0], 1, W, d, T, 0, 1, 1 << 30)
    assert v == [BEYOND] * 4 and total == 0 and st == ST_OVERFLOW and ap == {}
    v, total, st, ap = recover_batch(buf, offs[:3] + offs[:2], [0, 0, 0, 1, 1], 2, W, d, T, 0, 1, 2 * pitch(2))
    assert v == [ACC, ACC, ACC, STORE_FULL, STORE_FULL] and st == ST_STORE_FULL and list(ap) == [0]
    v, _, _, _ = recover_batch(buf, [offs[1], 0], [0, 5], 2, W, d, T, 0, 1, 1 << 30)
    assert v == [MALFORMED, MALFORMED]


def test_symbols_and_refusals_without_a_device():
    lib = _lib.load()
    assert lib.ss_follower_recover(None, None, 0, None, None, 0, None, 0, None, None) == _lib.SS_ERR_INVALID_ARG


# ---- GPU: the device call against the restatement -------------------------------------------------------------------
def _t(a, dt):
    import torch
    return torch.as_tensor(np.asarray(a), device="cuda:0").view(dt) if isinstance(a, np.ndarray) else torch.tensor(a, dtype=dt, device="cuda:0")


def _follower(ctx, G, n, me=0, W=64, mv=0, lv=1):
    """a fresh follower that remembers its DurEntry variants for the restatement"""
    from summerset_b200.engine import Follower
    f = Follower(ctx, G, n, me, window=W, meta_variant=mv, log_variant=lv)
    f.mv, f.lv = mv, lv
    return f


def _layout(recs, rng, align=None):
    """records at random offsets (or offset = k mod 16 when align is given) -> (bytes, offsets)"""
    buf, offs = bytearray(), []
    for k, r in enumerate(recs):
        if align is None:
            buf += bytes(rng.randint(0, 5))
        else:
            buf += bytes((align + k - len(buf)) % 16)
        offs.append(len(buf))
        buf += r
    return bytes(buf) + bytes(8), offs


_WORDS = ("start_slot", "log_end", "curr_term", "last_commit", "last_snap", "leader", "last_exec")
_RING = ("term", "shard_addr", "held", "data_len")
_VOTE = ("vote_term", "voted_for", "role_term", "role", "votes")


def _snap(fol):
    import torch
    torch.cuda.synchronize()
    s = {k: getattr(fol, k).cpu().numpy().copy() for k in _WORDS + _RING}
    vv = fol.vote_view()
    s.update({k: vv[k].cpu().numpy().copy() for k in _VOTE})
    return s


def recover_check(ctx, fol, recs, groups, rng, cap=None, pad=64, align=None, before=None):
    """one ss_follower_recover call on (record bytes, group) pairs, checked against the restatement: verdicts, total,
    status, every state word (the untouched ones equal to before the call), every shard through shard_addr with
    L..round16(L) zero, and the canary everywhere else.  Returns (verdicts, store tensor, applied)."""
    import torch
    d, T, W, G = fol.d, fol.T, fol.W, fol.G
    mv, lv = fol.mv, fol.lv
    buf, offs = _layout(recs, rng, align)
    _, total, _, _ = recover_batch(buf, offs, groups, G, W, d, T, mv, lv, 1 << 62)
    cap = total if cap is None else cap
    want_v, total, status, applied = recover_batch(buf, offs, groups, G, W, d, T, mv, lv, cap)
    before = _snap(fol) if before is None else before
    canary = np.frombuffer(rng.randbytes(pad + cap + pad), np.uint8).copy()
    full = torch.from_numpy(canary.copy()).cuda()
    store = full[pad:pad + max(cap, 16)]
    ctx.device_status()
    res = fol.recover(torch.from_numpy(np.frombuffer(buf, np.uint8).copy()).cuda(), _t(offs, torch.int64),
                      _t(np.array(groups, dtype=np.uint32), torch.int32), store, cap)
    torch.cuda.synchronize()
    assert [int(x) for x in res["verdict"].cpu().numpy().view(np.uint32)] == want_v
    assert int(res["total"][0]) == total
    assert ctx.device_status() == status
    after = _snap(fol)
    want = {k: v.copy() for k, v in before.items()}
    base = full.data_ptr() + pad
    st = full.cpu().numpy()
    written = np.zeros(len(st), dtype=bool)
    for g, (meta, ents, off) in applied.items():
        want["curr_term"][g] = np.int64(np.uint64(meta[1]).view(np.int64))
        want["vote_term"][g] = want["curr_term"][g]
        want["leader"][g], want["voted_for"][g] = NONE, meta[2]
        if not ents:
            continue
        start = int(before["start_slot"][g])
        want["log_end"][g] = start + len(ents)
        o = off
        for k in range(W):
            pos = (start + k) & (W - 1)
            if k >= len(ents):
                for a in _RING:
                    want[a][g, pos] = 0
                continue
            _, term, dl, shards = ents[k]
            held = sum(1 << j for j in shards)
            want["term"][g, pos] = np.uint64(term).view(np.int64)
            want["held"][g, pos], want["data_len"][g, pos] = np.uint32(held).view(np.int32), np.uint32(dl).view(np.int32)
            want["shard_addr"][g, pos] = base + o
            L = -(-dl // d)
            for r, j in enumerate(sorted(shards)):
                q = pad + o + r * pitch(L)
                assert st[q:q + L].tobytes() == shards[j], (g, k, j)
                assert not st[q + L:q + r16(L)].any(), (g, k, j)
                written[q:q + r16(L)] = True
            o += len(shards) * pitch(L)
    for k in want:
        assert np.array_equal(after[k], want[k]), k
    bad = np.nonzero((st != canary) & ~written)[0]
    assert len(bad) == 0, f"{len(bad)} store bytes outside the shards changed, first at {bad[0] - pad}"
    return want_v, full, applied


def _log(rng, d, T, n_ent, term=1, dls=(1, 10, 250), helds=None, lv=1, first_null=True):
    """a group's LogEntry records: the slot-0 null entry (when first_null), then n_ent entries"""
    recs = [null_record(d, T - d, lv)] if first_null else []
    full = (1 << T) - 1
    helds = helds or (1, full, (1 << d) - 1, 0)
    for k in range(n_ent - (1 if first_null else 0)):
        dl = dls[k % len(dls)]
        held = helds[k % len(helds)]
        recs.append(log_record(term + k // 3, d, T - d, dl, shards_of(rng, d, T, dl, held), bool(k & 1), k * 7, lv))
    return recs


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 5, 7, 16, 31, 32])
def test_populations_from_the_encoders(ctx, n):
    rng = random.Random(100 + n)
    d, T, G = n // 2 + 1, n, 6
    fol = _follower(ctx, G, n, n - 1)
    pairs = []
    for g in range(G):
        if g == 3:
            continue                                                          # a group with no records: untouched
        recs = [meta_record(g * 100 + 1, [0, n - 1, NONE, (n - 1) // 2][g % 4])] + _log(rng, d, T, 1 + 3 * g)
        pairs += [(g, r) for r in recs]
    per = {}
    for g, r in pairs:
        per.setdefault(g, []).append(r)
    order = []
    while any(per.values()):
        g = rng.choice([g for g in per if per[g]])
        order.append((g, per[g].pop(0)))
    v, _, _ = recover_check(ctx, fol, [r for _, r in order], [g for g, _ in order], rng)
    assert all(x == ACC for x in v)


@pytest.mark.gpu
@pytest.mark.parametrize("W", [2, 64, 4096])                             # 1: refused at creation
def test_windows_exactly_full_and_one_past(ctx, W):
    rng = random.Random(W)
    n, d = 3, 2
    fol = _follower(ctx, 3, n, 0, W)
    fol.start_slot[2] = 1000                                                  # a snapshot moved group 2's log start
    ok = [meta_record(5, 1)] + _log(rng, d, n, W, dls=(3,), helds=(1, 7))
    over = [meta_record(6, 2)] + _log(rng, d, n, W + 1, dls=(3,), helds=(1,))
    recs = ok + over + ok
    groups = [0] * len(ok) + [1] * len(over) + [2] * len(ok)
    v, _, _ = recover_check(ctx, fol, recs, groups, rng)
    assert v == [ACC] * len(ok) + [BEYOND] * len(over) + [ACC] * len(ok)
    assert int(fol.log_end[2]) == 1000 + W


@pytest.mark.gpu
@pytest.mark.parametrize("mv,lv", [(0, 250), (250, 0), (251, 65535), (65535, 251), (0, 1), (1, 0), (250, 251), (65535, 0)])
def test_variant_widths(ctx, mv, lv):
    rng = random.Random(mv * 7 + lv)
    n, d = 5, 3
    fol = _follower(ctx, 4, n, 2, 16, mv, lv)
    pairs = []
    for g in range(4):
        pairs += [(g, meta_record(g + 250, g, mv))] + [(g, r) for r in _log(rng, d, n, 4 + g, lv=lv)]
    # a record of the other variant in the LogEntry place ends group 3's log
    pairs.insert(len(pairs) - 2, (3, meta_record(9, 0, mv)))
    v, _, _ = recover_check(ctx, fol, [r for _, r in pairs], [g for g, _ in pairs], rng)
    assert v[-3:] == [MALFORMED, AFTER_END, AFTER_END]


@pytest.mark.gpu
@pytest.mark.parametrize("align", [None] + list(range(16)))
def test_terms_votes_offsets_and_shard_lengths(ctx, align):
    """curr_term and entry terms at every varint width, voted_for 0 / me / n - 1 / None, non-minimal varints, records at
    every offset mod 16 (align) or at random ones with shard lengths 1, 15-17, 250, 251, 65535 and 65536; empty,
    single, full and 0..majority held masks"""
    rng = random.Random(5 if align is None else 50 + align)
    n, d, me = 5, 3, 2
    terms = [0, 250, 251, 1 << 16, (1 << 32) - 1, 1 << 32, (1 << 64) - 1]
    votes = [0, me, n - 1, NONE]
    sls = [1, 15, 16, 17] if align is not None else [1, 15, 16, 17, 250, 251, 65535, 65536]
    helds = [0, 1 << 4, 31, 7]
    fol = _follower(ctx, len(terms), n, me, 16)
    pairs = []
    for g, t in enumerate(terms):
        if g == 1:                                                   # curr_term 250 as a non-minimal u32 varint
            pairs.append((g, framed(b"\x00\xfc" + (250).to_bytes(4, "little") + bytes([votes[1]]))))
        else:
            pairs.append((g, meta_record(t, votes[g % 4])))
        for k in range(4):
            L = sls[(g * 4 + k) % len(sls)]
            dl = L * d - (k % d)
            held = helds[(g + k) % 4]
            sh = shards_of(rng, d, n, dl, held)
            if k == 1:                                               # data_len as a non-minimal u64 varint
                rest = tf.codeword(d, n - d, dl, sh)[2 + len(vi(dl)):]
                rec = framed(vi(1) + vi(t) + bytes([d, n - d]) + b"\xfd" + dl.to_bytes(8, "little") + rest + b"\x00" + vi(0))
            else:
                rec = log_record(t, d, n - d, dl, sh, bool(k & 1), t)
            pairs.append((g, rec))
    v, _, _ = recover_check(ctx, fol, [r for _, r in pairs], [g for g, _ in pairs], rng, align=align)
    assert all(x == ACC for x in v)


@pytest.mark.gpu
def test_log_ends(ctx):
    """each malformed rule ends its group's log: the records before apply, the later ones get AFTER_END"""
    rng = random.Random(11)
    n, d, T = 5, 3, 5
    G = 12
    fol = _follower(ctx, G, n, 0, 16)
    good = lambda: log_record(3, d, T - d, 7, shards_of(rng, d, T, 7, 5))
    g0 = good()
    bad = [
        g0[:-3],                                                              # a partial tail (the buffer ends below)
        framed(g0[8:] + b"\x00"),                                             # trailing bytes
        log_record(3, d, T - d, 7, {}, variant=2),                            # a foreign variant
        log_record(3, 2, T - 2, 7, {}),                                       # the wrong code
        framed(vi(1) + vi(3) + bytes([d, T - d]) + vi(7) + vi(4) + vi(T) + b"\x00" * T + b"\x00\x00" + vi(0)),   # shard_len
        framed(vi(1) + vi(3) + bytes([d, T - d]) + vi(7) + vi(3) + vi(T) + b"\x01" + vi(2) + b"ab" + b"\x00" * (T - 1) + b"\x00\x00" + vi(0)),
        framed(vi(1) + vi(3) + tf.codeword(d, T - d, 7, {})[:-1] + b"\x01" + vi(7) + bytes(7) + b"\x00" + vi(0)),   # data_copy Some
        framed(vi(1) + vi(3) + tf.codeword(d, T - d, 7, {}) + b"\x02" + vi(0)),                                 # external 2
        meta_record(4, 1),                                                    # a second Metadata
    ]
    pairs = []
    for g, b in enumerate(bad[1:], start=1):
        pairs += [(g, meta_record(2, 0)), (g, null_record(d, T - d)), (g, good()), (g, b), (g, good()), (g, meta_record(9))]
    pairs += [(10, good()), (10, meta_record(3))]                              # Metadata not first
    pairs += [(G + 3, meta_record(1)), (G, good())]                           # groups >= G
    pairs += [(0, meta_record(2, 0)), (0, good()), (0, bad[0])]               # the partial tail last in the buffer
    recs, groups = [r for _, r in pairs], [g for g, _ in pairs]
    buf, offs = _layout(recs, rng)
    buf = buf[:offs[-1] + len(bad[0])]                                        # ... cut at its end
    import torch
    want = recover_batch(buf, offs, groups, G, 16, d, T, 0, 1, 1 << 40)
    assert want[0][-1] == MALFORMED and want[0][-3:-1] == [ACC, ACC]
    for g in range(1, len(bad)):
        assert want[0][6 * (g - 1):6 * g] == [ACC, ACC, ACC, MALFORMED, AFTER_END, AFTER_END], g
    assert want[0][6 * (len(bad) - 1):6 * (len(bad) - 1) + 4] == [MALFORMED, AFTER_END, MALFORMED, MALFORMED]
    before = _snap(fol)
    store = torch.zeros(want[1] + 64, dtype=torch.uint8, device="cuda:0")
    res = fol.recover(torch.from_numpy(np.frombuffer(buf, np.uint8).copy()).cuda(), _t(offs, torch.int64),
                      _t(np.array(groups, dtype=np.uint32), torch.int32), store)
    torch.cuda.synchronize()
    assert [int(x) for x in res["verdict"].cpu().numpy().view(np.uint32)] == want[0]
    assert ctx.device_status() == 0
    after = _snap(fol)
    assert int(after["log_end"][0]) == 1 and int(after["term"][0, 0]) == 3 and int(after["curr_term"][10]) == 0 and int(after["log_end"][10]) == 1
    for g in range(1, len(bad)):
        assert int(after["log_end"][g]) == 2 and int(after["curr_term"][g]) == 2 and int(after["voted_for"][g]) == 0
    assert np.array_equal(after["term"][11], before["term"][11])


@pytest.mark.gpu
def test_store_cut_at_every_group_boundary(ctx):
    rng = random.Random(12)
    n, d, G = 3, 2, 5
    logs = {g: [meta_record(g + 1, g % 3)] + _log(rng, d, n, 2 + g, dls=(5, 40)) for g in range(G)}
    pairs = [(g, r) for g in range(G) for r in logs[g]]
    recs, groups = [r for _, r in pairs], [g for g, _ in pairs]
    one = _follower(ctx, G, n, 1, 16)
    _, store_one, _ = recover_check(ctx, one, recs, groups, rng)
    want = _snap(one)
    ends = np.cumsum([sum(ent_bytes(parse_record(r, 0, d, n, 0, 1), d) for r in logs[g][1:]) for g in range(G)])
    for b in range(G):
        for cap in (int(ends[b]), int(ends[b]) + 1, int(ends[b + 1]) - 1 if b + 1 < G else None):
            if cap is None:
                continue
            fol = _follower(ctx, G, n, 1, 16)
            v, s1, ap = recover_check(ctx, fol, recs, groups, rng, cap=cap)
            assert sorted(ap) == list(range(b + 1)) and (b == G - 1 or STORE_FULL in v)
            rest = [i for i, x in enumerate(v) if x == STORE_FULL]
            if rest:
                recover_check(ctx, fol, [recs[i] for i in rest], [groups[i] for i in rest], rng)
            got = _snap(fol)
            for k in want:
                if k == "shard_addr":
                    continue
                assert np.array_equal(got[k], want[k]), (b, cap, k)


@pytest.mark.gpu
def test_edges_grid_caps_sort_keys_and_one_long_group(ctx):
    import torch
    rng = random.Random(13)
    n, d = 3, 2
    # one group of 4097 records: the Metadata and 4096 entries at window 4096
    fol = _follower(ctx, 1, n, 0, 4096)
    recs = [meta_record(7, 0)] + _log(rng, d, n, 4096, dls=(1, 2), helds=(1, 2, 4))
    recover_check(ctx, fol, recs, [0] * len(recs), rng)
    # G at the sort-key edges: every group one Metadata and one entry, in reverse group order
    for G in (1, 255, 256, 257, 65535, 65536, 65537):
        fol = _follower(ctx, G, n, 0, 2)
        e = log_record(1, d, 1, 3, {0: b"xy"})
        m = meta_record(3, 1)
        k = min(G, 300)
        gs = sorted(set([0, G - 1] + rng.sample(range(G), k)), reverse=True)
        recs, groups = [], []
        for g in gs:
            recs += [m, e]
            groups += [g, g]
        v, _, _ = recover_check(ctx, fol, recs, groups, rng) if G <= 257 else (None, None, None)
        if v is None:                                                       # large G: only the words, no restatement walk
            buf, offs = _layout(recs, rng)
            st = torch.zeros(len(gs) * 32 + 16, dtype=torch.uint8, device="cuda:0")
            res = fol.recover(torch.from_numpy(np.frombuffer(buf, np.uint8).copy()).cuda(), _t(offs, torch.int64),
                              _t(np.array(groups, dtype=np.uint32), torch.int32), st)
            torch.cuda.synchronize()
            assert (res["verdict"].cpu().numpy().view(np.uint32) == ACC).all() and int(res["total"][0]) == 32 * len(gs)
            le = fol.log_end.cpu().numpy()
            assert (le[gs] == 1).all() and int(fol.curr_term[G - 1]) == 3
            addr = fol.shard_addr[:, 0].cpu().numpy()[gs[::-1]] - st.data_ptr()
            assert (addr == 32 * np.arange(len(gs))).all()
        assert ctx.device_status() == 0
    # past every kernel's grid cap: a thread per record or segment, a warp per applied entry
    warps, threads = ctx.sm_count * 64 * 8, ctx.sm_count * 64 * 256
    G = warps + 100
    fol = _follower(ctx, G, n, 0, 2)
    e, m = log_record(1, d, 1, 3, {1: b"zz"}), meta_record(4, 2)
    X = threads + 100 - 2 * G
    recs = [m, e] * G + [m] * X
    groups = np.concatenate([np.repeat(np.arange(G), 2), np.full(X, G + 1)]).astype(np.uint32)
    cell = 32
    buf = np.zeros(cell * len(recs) + 16, dtype=np.uint8)
    offs = 1 + cell * np.arange(len(recs), dtype=np.int64)
    for k, r in enumerate((m, e)):
        sel = offs[:2 * G][k::2]
        buf[sel[:, None] + np.arange(len(r))] = np.frombuffer(r, np.uint8)
    buf[offs[2 * G:][:, None] + np.arange(len(m))] = np.frombuffer(m, np.uint8)
    full = torch.full((G * 32 + 128,), 0xA5, dtype=torch.uint8, device="cuda:0")
    res = fol.recover(torch.from_numpy(buf).cuda(), torch.from_numpy(offs).cuda(), torch.from_numpy(groups.view(np.int32)).cuda(),
                      full[64:64 + G * 32])
    torch.cuda.synchronize()
    v = res["verdict"].cpu().numpy().view(np.uint32)
    assert (v[:2 * G] == ACC).all() and (v[2 * G:] == MALFORMED).all() and int(res["total"][0]) == G * 32
    st = full.cpu().numpy()
    assert (st[:64] == 0xA5).all() and (st[64 + G * 32:] == 0xA5).all()
    want = np.full(32, 0xA5, np.uint8)
    want[:16] = 0
    want[:2] = np.frombuffer(b"zz", np.uint8)
    assert (st[64:64 + G * 32].reshape(G, 32) == want).all()
    assert (fol.log_end.cpu().numpy() == 1).all() and (fol.vote_view()["voted_for"].cpu().numpy() == 2).all()
    assert ctx.device_status() == 0


@pytest.mark.gpu
def test_scratch_regrown_and_reused_empty_batch_and_refusals(ctx):
    import torch
    rng = random.Random(14)
    n, d = 3, 2
    fol = _follower(ctx, 4, n, 0, 8)
    small = [meta_record(1)] + _log(rng, d, n, 2)
    recover_check(ctx, fol, small, [1] * len(small), rng)
    big = [meta_record(2, 1)] + _log(rng, d, n, 8)
    recover_check(ctx, fol, big * 1 + small, [2] * len(big) + [3] * len(small), rng)   # the scratch grows
    recover_check(ctx, fol, small, [0] * len(small), rng)                              # and is reused
    lib = fol.lib
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    m = meta_record(9, 0)
    buf[:len(m)] = torch.tensor(list(m), dtype=torch.uint8)
    off, grp = torch.zeros(1, dtype=torch.int64, device="cuda:0"), torch.zeros(1, dtype=torch.int32, device="cuda:0")
    store = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    verdict = torch.full((1,), 7, dtype=torch.int32, device="cuda:0")
    total = torch.full((1,), 7, dtype=torch.int64, device="cuda:0")
    p = lambda x: x.data_ptr()

    def call(f=fol, n_=1, b=p(buf), o=p(off), g=p(grp), s=p(store), v=p(verdict), t=p(total)):
        return lib.ss_follower_recover(f.h, b, 64, o, g, n_, s, 64, v, t)

    before = _snap(fol)
    bad = _lib.SS_ERR_INVALID_ARG
    for k in ("b", "o", "g", "s", "v"):
        assert call(**{k: None}) == bad, k
    assert call(s=p(store) + 8) == bad
    assert call(n_=1 << 31) == bad
    same = _follower(ctx, 4, n, 0, 8, 3, 3)
    assert call(f=same) == bad and call(f=same, n_=0) == bad                           # equal variants
    torch.cuda.synchronize()
    assert int(verdict[0]) == 7 and int(total[0]) == 7 and ctx.device_status() == 0
    after = _snap(fol)
    assert all(np.array_equal(before[k], after[k]) for k in before)
    assert call(n_=0) == _lib.SS_OK and int(total[0]) == 0
    assert lib.ss_follower_recover(fol.h, None, 0, None, None, 0, None, 0, None, None) == _lib.SS_OK
    assert call(t=None) == _lib.SS_OK
    torch.cuda.synchronize()
    assert int(verdict[0]) == ACC - (1 << 32) and int(fol.curr_term[0]) == 9 and int(fol.leader[0]) == NONE


# ---- GPU: the round trip from a live cluster -----------------------------------------------------------------------
class Wal:
    """each replica's WAL per group as its host keeps it: the Metadata record at the head (rewritten in place), then
    the LogEntry records, the slot-0 null entry first; a Truncate cuts the records from the truncated slot on"""

    def __init__(self, n, G):
        d = n // 2 + 1
        self.recs = {r: {g: [meta_record(0), null_record(d, n - d)] for g in range(G)} for r in range(n)}

    def meta(self, r, groups, out):
        ml, cells = out["meta_len"].cpu().tolist(), out["meta"].cpu().numpy()
        for i, g in enumerate(groups):
            if ml[i]:
                self.recs[r][g][0] = cells[i][:ml[i]].tobytes()

    def records(self, r, g, wal, off, ln):
        end = off + ln
        while off < end:
            k = int.from_bytes(wal[off:off + 8].tobytes(), "big")
            self.recs[r][g].append(wal[off:off + 8 + k].tobytes())
            off += r16(8 + k)

    def append(self, r, groups, a, wal):
        w = wal.cpu().numpy()
        for i, g in enumerate(groups):
            ts_, wl = int(a["trunc_slot"][i]), int(a["wal_len"][i])
            if ts_ >= 0:
                del self.recs[r][g][1 + ts_:]
            if wl:
                self.records(r, g, w, int(a["wal_off"][i]), wl)
        self.meta(r, groups, a)

    def propose(self, r, o, wal):
        w = wal.cpu().numpy()
        for g, (wo, wl) in enumerate(zip(o["wal_off"].cpu().tolist(), o["wal_len"].cpu().tolist())):
            if wo >= 0 and wl:
                self.records(r, g, w, wo, wl)

    def batch(self, r, rng):
        """the replica's records, groups interleaved at random with each group's order kept"""
        per = {g: list(x) for g, x in self.recs[r].items()}
        out = []
        while any(per.values()):
            g = rng.choice([g for g in per if per[g]])
            out.append((g, per[g].pop(0)))
        return [x for _, x in out], [g for g, _ in out]


def _prop(eng, me, lens, stride, keep, batch, rng, full_copy, wal_log):
    import torch
    from tests import test_craft_stepup as ts
    bs = [rng.randbytes(x) for x in lens]
    arena, offs = bytearray(), []
    for b in bs:
        offs.append(len(arena))
        arena += b
    store = torch.zeros((eng.P + 1, stride), dtype=torch.uint8, device="cuda:0")
    keep.append(store)
    wal = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
    o = eng.propose(me, ts._t(np.frombuffer(bytes(arena) + b"\0", dtype=np.uint8), torch.uint8), ts._t(offs, torch.int64),
                    ts._t(lens, torch.int32), store, wal, full_copy=full_copy)
    torch.cuda.synchronize()
    wal_log.propose(me, o, wal)
    out = {}
    for g, (x, s) in enumerate(zip(lens, o["slot_out"].cpu().tolist())):
        if x:
            out[(g, s)] = bs[g]
    batch.update(out)
    return out


def _rep(ctx, eng, me, fols, keep, rng, full_copy, wal_log, heartbeat_only=False):
    """tests/test_craft_stepdown.py's replication round with every follower's records and cells kept in wal_log"""
    import torch
    from summerset_b200.engine import append_reply_parse
    from tests import test_craft_stepup as ts
    dev = "cuda:0"
    for heartbeat in ((True,) if heartbeat_only else (False, True)):
        out = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
        o = eng.pack_append(me, out, 1 << 12, heartbeat=heartbeat, msg_chunk_size=4, full_copy=full_copy)
        torch.cuda.synchronize()
        nf = int(o["n_frames"][0])
        fo, fg, fp = o["frame_off"][:nf], o["frame_group"][:nf], o["frame_peer"][:nf]
        replies = []
        for r, f in fols.items():
            q = r if r < me else r - 1
            sel = (fp == q).nonzero().flatten()
            if sel.numel() == 0:
                continue
            st = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
            keep.append(st)
            wal = torch.zeros(1 << 22, dtype=torch.uint8, device=dev)
            a = f.append(out, fo[sel].contiguous(), fg[sel].contiguous(), torch.full_like(fp[sel], me), st, wal)
            torch.cuda.synchronize()
            assert (a["verdict"].cpu().numpy().view(np.uint32) == tf.ACCEPTED).all()
            groups = fg[sel].cpu().tolist()
            wal_log.append(r, groups, a, wal)
            rl, cells = a["reply_len"].cpu().numpy(), a["replies"].cpu().numpy()
            replies += [(g, q, cells[i][:rl[i]].tobytes()) for i, g in enumerate(groups)]
        if replies:
            tb, offs = ts._buf([x for _, _, x in replies], rng)
            rec = append_reply_parse(ctx, tb, ts._t(offs, torch.int64), ts._t([x[0] for x in replies], torch.int32),
                                     ts._t([x[1] for x in replies], torch.uint8), eng.curr_term, eng.G)
            eng.on_append_replies(rec["rec_group"], rec["rec_peer"], rec["rec_end_slot"])
            eng.tick()
            torch.cuda.synchronize()


def _elect(ctx, fols, cand, voters, G, source, rng, wal_log):
    import torch
    from tests import test_craft_election as te
    from tests import test_craft_stepup as ts
    groups = list(range(G))
    c = fols[cand].campaign(ts._t(groups, torch.int32), ts._t([source] * G, torch.uint8))
    torch.cuda.synchronize()
    assert (c["verdict"].cpu().numpy() == te.DONE).all()
    wal_log.meta(cand, groups, c)
    fl, fr = c["frame_len"].cpu().tolist(), c["frames"].cpu().numpy()
    replies = []
    for v in voters:
        r_ = te._deliver(fols[v], [(g, cand, fr[g][:fl[g]].tobytes()) for g in groups], rng, "vote")
        assert (r_["verdict"].cpu().numpy().view(np.uint32) == te.GRANTED).all()
        wal_log.meta(v, groups, r_)
        rl, cells = r_["reply_len"].cpu().tolist(), r_["replies"].cpu().numpy()
        replies += [(g, v, cells[g][:rl[g]].tobytes()) for g in groups]
    t = te._deliver(fols[cand], replies, rng, "tally")
    wal_log.meta(cand, [g for g, _, _ in replies], t)
    assert int(t["n_won"][0]) == G
    return t


def _exec(x):
    import torch
    out = torch.zeros(1 << 23, dtype=torch.uint8, device="cuda:0")
    ex = x.execute(out, 1 << 14)
    torch.cuda.synchronize()
    o_ = out.cpu().numpy()
    return [((g, s), o_[off:off + dl].tobytes())
            for g, s, off, dl in zip(*(ex[k][:int(ex["totals"][0])].cpu().tolist() for k in ("rec_group", "rec_slot", "rec_off", "rec_len")))]


def _dev_bytes(addr, nb):
    """nb bytes of device memory at addr, as a numpy array"""
    import torch
    from summerset_b200.engine import _DevArray
    return torch.as_tensor(_DevArray(addr, (nb,), "|u1"), device="cuda:0").cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("full_copy", [True, False])
@pytest.mark.parametrize("n", [3, 5, 7])
def test_round_trip_from_a_live_cluster(ctx, n, full_copy):
    """replica 0 leads, commits and keeps a suffix to itself; replica 1 is elected, steps up, deposes replica 0 and
    truncates that suffix.  Every replica's WAL is replayed into a fresh follower: the state must equal the live
    follower's (held shards: the durable ones, byte for byte the live follower's), and the recovered followers vote,
    campaign, commit, execute and step up as the live ones do"""
    import torch
    from summerset_b200.engine import RaftEngine
    from tests import test_craft_election as te
    from tests import test_craft_leader as tl
    from tests import test_craft_stepup as ts
    G, W = 12, 64
    d = n // 2 + 1
    rng = random.Random(5500 + n + full_copy)
    wl = Wal(n, G)
    fols = {r: _follower(ctx, G, n, r, W) for r in range(n)}
    stride = G * tl.pitch(-(-3000 // d)) * 8
    keep, batch, committed = [], {}, {}
    lens = lambda: [rng.choice((0, 1, 17, 300, 3000)) for _ in range(G)]
    e0 = RaftEngine(ctx, G, n, craft=True, window=W)
    e0.set_full_copy(full_copy)
    e0.log_view()
    e0.curr_term.fill_(1)
    for _ in range(2):
        committed.update(_prop(e0, 0, lens(), stride, keep, batch, rng, full_copy, wl))
        _rep(ctx, e0, 0, {r: f for r, f in fols.items() if r}, keep, rng, full_copy, wl)
    lost = _prop(e0, 0, [x or 5 for x in lens()], stride, keep, batch, rng, full_copy, wl)   # never leaves replica 0
    t = _elect(ctx, fols, 1, range(2, n), G, 0, rng, wl)
    e1 = RaftEngine(ctx, G, n, craft=True, window=W)
    e1.set_full_copy(full_copy)
    e1.recon_view(), e1.log_view()
    p1 = torch.zeros((n, stride), dtype=torch.uint8, device="cuda:0")
    keep.append(p1)
    su = e1.step_up(fols[1], t["won_group"], t["won_term"], p1)
    torch.cuda.synchronize()
    assert (su["verdict"].cpu().numpy() == ts.DONE).all()
    out = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
    hb = e1.pack_append(1, out, 1 << 12, heartbeat=True, full_copy=full_copy)
    torch.cuda.synchronize()
    nf = int(hb["n_frames"][0])
    sel = (hb["frame_peer"][:nf] == 0).nonzero().flatten()
    store0 = torch.zeros(1 << 24, dtype=torch.uint8, device="cuda:0")
    keep.append(store0)
    sg = hb["frame_group"][sel].contiguous()
    sd = e0.step_down(fols[0], out, hb["frame_off"][sel].contiguous(), sg, torch.ones(sel.numel(), dtype=torch.uint8, device="cuda:0"),
                      store0)
    torch.cuda.synchronize()
    wl.meta(0, sg.cpu().tolist(), sd)
    committed.update(_prop(e1, 1, [x or 5 for x in lens()], stride, keep, batch, rng, full_copy, wl))
    _rep(ctx, e1, 1, {r: f for r, f in fols.items() if r != 1}, keep, rng, full_copy, wl)
    for (g, s) in lost:                                  # replica 0's suffix was truncated and replaced in its WAL
        assert len(wl.recs[0][g]) == 2 + s and parse_record(wl.recs[0][g][1 + s], 0, d, n, 0, 1)[1] == 2, (g, s)
    # every replica's WAL into a fresh follower
    rec = {}
    for r in range(n):
        recs, groups = wl.batch(r, rng)
        f = _follower(ctx, G, n, r, W)
        v, store, applied = recover_check(ctx, f, recs, groups, rng)
        assert all(x == ACC for x in v)
        keep.append(store)
        rec[r] = f
        live, got = _snap(fols[r]), _snap(f)
        # replica 1 leads: its own entries are in its engine's log and its WAL, not in its live follower
        want_end = e1.log_end.cpu().numpy() if r == 1 else live["log_end"]
        assert np.array_equal(got["log_end"], want_end), r
        for k in ("curr_term", "start_slot"):
            assert np.array_equal(live[k], got[k]), (r, k)
        ct = live["curr_term"]
        vf = np.where(live["vote_term"] == ct, live["voted_for"], NONE)
        assert np.array_equal(vf, got["voted_for"]) and np.array_equal(got["vote_term"], ct), r
        for g in range(G):
            for s in range(int(live["log_end"][g])):
                pos = s & (W - 1)
                assert live["term"][g, pos] == got["term"][g, pos] and live["data_len"][g, pos] == got["data_len"][g, pos], (r, g, s)
                hl, hg = int(live["held"][g, pos]), int(got["held"][g, pos])
                assert hg & ~hl == 0, (r, g, s)               # the durable shards are held live too
                L = -(-int(live["data_len"][g, pos]) // d)
                for j in range(n):
                    if (hg >> j) & 1:
                        a = int(live["shard_addr"][g, pos]) + bin(hl & ((1 << j) - 1)).count("1") * pitch(L)
                        b = int(got["shard_addr"][g, pos]) + bin(hg & ((1 << j) - 1)).count("1") * pitch(L)
                        assert np.array_equal(_dev_bytes(a, L), _dev_bytes(b, L)), (r, g, s, j)
    # RequestVote at the recovered term: a second candidate is refused, the one voted for is granted again
    for r in range(2, n):
        ct = int(rec[r].curr_term[0])
        le = int(rec[r].log_end[0])
        lt = int(rec[r].term[0, (le - 1) & (W - 1)])
        x = te._deliver(rec[r], [(0, n - 1 if r != n - 1 else 0, te.request_vote(ct, le + 5, lt)),
                                 (0, 1, te.request_vote(ct, le + 5, lt))], rng, "vote")
        assert x["verdict"].cpu().numpy().view(np.uint32).tolist() == [te.NO_REPLY, te.GRANTED]
    # campaign on recovered replica 0: its RequestVote carries the recovered last_slot / last_term
    c = rec[0].campaign(ts._t([3], torch.int32))
    torch.cuda.synchronize()
    le, tm = int(fols[0].log_end[3]), int(fols[0].term[3, (int(fols[0].log_end[3]) - 1) & (W - 1)])
    assert c["frames"][0][:int(c["frame_len"][0])].cpu().numpy().tobytes() == framed(vi(0) + vi(2) + vi(int(fols[0].curr_term[3]) + 1) + vi(le - 1) + vi(tm))
    if full_copy:
        # the leader's heartbeat commits the recovered log; execution delivers the committed payloads
        out = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
        hb = e1.pack_append(1, out, 1 << 12, heartbeat=True, full_copy=True)
        torch.cuda.synchronize()
        nf = int(hb["n_frames"][0])
        seq = sorted(committed)
        for r in range(2, n):
            q = r - 1
            sel = (hb["frame_peer"][:nf] == q).nonzero().flatten()
            st = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
            a = rec[r].append(out, hb["frame_off"][sel].contiguous(), hb["frame_group"][sel].contiguous(),
                              torch.full((sel.numel(),), 1, dtype=torch.uint8, device="cuda:0"), st, torch.zeros(1 << 20, dtype=torch.uint8, device="cuda:0"))
            torch.cuda.synchronize()
            assert (a["verdict"].cpu().numpy().view(np.uint32) == tf.ACCEPTED).all()
            ran = _exec(rec[r])
            assert sorted(k for k, _ in ran) == seq and all(v == committed[k] for k, v in ran), r
            assert ran == _exec_live(fols[r], e1, r, ctx, rng, keep)
    # step-up takes the recovered log
    e2 = RaftEngine(ctx, G, n, craft=True, window=W)
    e2.set_full_copy(full_copy)
    e2.recon_view(), e2.log_view()
    p2 = torch.zeros((n, stride), dtype=torch.uint8, device="cuda:0")
    keep.append(p2)
    r = n - 1
    terms = rec[r].curr_term.clone() + 1
    su = e2.step_up(rec[r], torch.arange(G, dtype=torch.int32, device="cuda:0"), terms, p2)
    torch.cuda.synchronize()
    assert (su["verdict"].cpu().numpy() == ts.DONE).all()
    assert e2.log_end.cpu().tolist() == rec[r].log_end.cpu().tolist()
    for x in (e0, e1, e2):
        x.close()
    for f in list(fols.values()) + list(rec.values()):
        f.close()


def _exec_live(fol, eng, r, ctx, rng, keep):
    """the live follower, given the same heartbeat, executes the same payloads"""
    import torch
    out = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
    hb = eng.pack_append(1, out, 1 << 12, heartbeat=True, full_copy=True)
    torch.cuda.synchronize()
    nf = int(hb["n_frames"][0])
    sel = (hb["frame_peer"][:nf] == r - 1).nonzero().flatten()
    st = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda:0")
    keep.append(st)
    fol.append(out, hb["frame_off"][sel].contiguous(), hb["frame_group"][sel].contiguous(),
               torch.full((sel.numel(),), 1, dtype=torch.uint8, device="cuda:0"), st, torch.zeros(1 << 20, dtype=torch.uint8, device="cuda:0"))
    torch.cuda.synchronize()
    return _exec(fol)
