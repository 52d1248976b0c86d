"""The leader's Accept / WAL AcceptData frame packers across what their ABI accepts:

  ss_frame_accept_pack_dev         frame_pack_kernel (wire_kernels.cu): the general packer, uniform codewords
  ss_frame_accept_batch_dev        frame_accept_kernel (tally_kernels.cu): the single-shard fast path
  ss_frame_accept_pack_ragged_dev  frame_size_ragged_kernel + scan + frame_pack_ragged_kernel
  ss_frame_accept_max_len          the host bound callers size frame slots with

Expected bytes come from oracle/ss_wire.c (ssor_frame_accept / ssor_wal_accept_data), never from product code; every
produced frame also goes through the oracle's decoder and must decode to what went in.  Every output buffer starts as
0xA5 and every byte outside the frames must still be 0xA5 afterwards.  The library is called through ctypes wherever
summerset_b200.api pins an argument (assign_size, strides, frame_stride, a NULL policy_idx).

  1-3   (no device) the three length bounds against the longest frames the oracle can build
  4     general packer: code x population x peer x kind, every shape of policy row, out-of-range and NULL policy_idx
  5     shard lengths at the varint and vector-copy edges, 1 / 2 / T shards per frame, wide shard and plane strides
  6     msg_variant, slot, ballot, assign_size and policy-row varint widths
  7     frames that fit their slot beside frames that do not
  8     batches past the launch's grid cap, two calls back to back
  9     the fast path: codes up to T = 250, shard_idx beyond a warp, exact and wide strides
  10    the three packers against each other; the ragged packer called raw
  11    refusals
"""
import ctypes as C

import numpy as np
import pytest
import torch

from summerset_b200 import _lib
from summerset_b200.api import frame_accept_room, round_up

DEV = "cuda:0"
PAT = 0xA5
OFF_PAT, LEN_PAT = -0x0123456789ABCDF0, 0x5A5A5A5A         # frame_off / frame_len before a call
U32MAX, U64MAX = (1 << 32) - 1, (1 << 64) - 1
PEER, WAL = 0, 1                                            # SS_FRAME_PEER_ACCEPT / SS_FRAME_WAL_ACCEPT_DATA
INVALID = _lib.SS_ERR_INVALID_ARG
OVERFLOW = 4                                                # SS_DEV_STATUS_FRAME_OVERFLOW
SPECIAL = [0, 1, 250, 251, 252, 65535, 65536, U32MAX, 1 << 32, (1 << 63) + 5, U64MAX]     # every varint boundary
VARIANTS = [0, 2, 250, 251, 65535, 65536, U32MAX]
L_EDGES = [1, 2, 15, 16, 17, 31, 32, 33, 249, 250, 251, 252, 4095, 4096, 4097, 65535, 65536, 65537]
KINDS = {"rspaxos_accept": (PEER, False), "crossword_accept": (PEER, True), "wal_accept_data": (WAL, False)}


def _t(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a).to(DEV)


def _vlen(a):
    """bytes of a bincode varint (pinned to oracle.varint by test_helpers_agree_with_the_oracle)"""
    a = np.asarray(a, dtype=np.uint64)
    return 1 + 2 * (a >= 251).astype(np.int64) + 2 * (a >= 1 << 16) + 4 * (a >= 1 << 32)


def _slots_ballots(rng, n):
    """every pair of varint boundaries in the first 121 frames, random values after"""
    i = np.arange(n)
    sp = np.array(SPECIAL, dtype=np.uint64)
    slot = np.where(i < 121, sp[i % 11], rng.integers(0, 1 << 40, n).astype(np.uint64))
    ballot = np.where(i < 121, sp[i // 11 % 11], rng.integers(0, 1 << 20, n).astype(np.uint64))
    return slot.astype(np.uint64), ballot.astype(np.uint64)


class _Wire:
    """oracle/ss_wire.c's encoder and decoder, called on shard bytes where they lie in host memory and with the shard
    length stated, so that a frame carrying no shard has expected bytes too"""

    def __init__(self, oracle):
        self.lib = oracle.lib()
        self.lib.ssor_frame_accept.restype = C.c_size_t
        self.lib.ssor_wal_accept_data.restype = C.c_size_t
        self.lib.ssor_decode_accept.restype = C.c_long
        self.buf = np.zeros(1 << 16, dtype=np.uint8)

    def encode(self, kind, variant, slot, ballot, d, p, dlen, L, ptrs, asg=None, asz=0):
        """ptrs: d + p host addresses (0 = None).  asg: the policy row (assignment: Vec<Bitmap>) or None."""
        need = 256 + (d + p) + sum(1 for q in ptrs if q) * (L + 8) + (16 * len(asg) if asg is not None else 0)
        if need > self.buf.size:
            self.buf = np.zeros(2 * need, dtype=np.uint8)
        arr = (C.c_void_p * (d + p))(*[q or None for q in ptrs])
        out = C.c_void_p(self.buf.ctypes.data)
        if kind == WAL and variant == 1 and asg is None:
            n = self.lib.ssor_wal_accept_data(C.c_uint64(slot), C.c_uint64(ballot), d, p, C.c_uint64(dlen), C.c_uint64(L), arr, out)
            return self.buf[:n].tobytes()
        a = None if asg is None else np.ascontiguousarray(asg, dtype=np.uint32)
        n = self.lib.ssor_frame_accept(C.c_uint32(variant), C.c_uint64(slot), C.c_uint64(ballot), d, p, C.c_uint64(dlen), C.c_uint64(L),
                                       arr, None if a is None else C.c_void_p(a.ctypes.data), 0 if a is None else len(a), asz, out)
        fr = self.buf[:n].tobytes()
        if kind == WAL:
            # a WalEntry is not wrapped in PeerMessage::Msg: the same body less its first byte (pinned against
            # ssor_wal_accept_data by test_helpers_agree_with_the_oracle)
            fr = (len(fr) - 9).to_bytes(8, "big") + fr[9:]
        return fr

    def decode(self, frame, kind, with_asg):
        buf = np.frombuffer(frame, dtype=np.uint8)
        variant, d, p, n_asg, asz = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
        slot, ballot, dl, sl = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        at = np.zeros(256, dtype=np.uint64)
        asg = np.zeros(64, dtype=np.uint32)
        n = self.lib.ssor_decode_accept(C.c_void_p(buf.ctypes.data), C.c_size_t(len(frame)), kind, C.byref(variant), C.byref(slot),
                                        C.byref(ballot), C.byref(d), C.byref(p), C.byref(dl), C.byref(sl), C.c_void_p(at.ctypes.data), 256,
                                        1 if with_asg else 0, C.c_void_p(asg.ctypes.data), C.byref(n_asg), C.byref(asz))
        if n < 0:
            return None
        return dict(length=int(n), variant=variant.value, slot=slot.value, ballot=ballot.value, d=d.value, p=p.value,
                    data_len=dl.value, shard_len=sl.value, at=[int(x) for x in at[:d.value + p.value]],
                    assignment=[int(x) for x in asg[:n_asg.value]] if with_asg else None, assign_size=asz.value)


@pytest.fixture(scope="module")
def wire(oracle):
    return _Wire(oracle)


class _Batch:
    """n uniform codewords of one code as the packers take them: random shard planes (bytes [L, round_up(L, 16)) of a
    slot zero, whatever lies between the slots random), slots, ballots, a policy table -- and the oracle's frame for
    every codeword"""

    def __init__(self, rng, d, T, data_len, n, pop, policies, pidx, kind=PEER, variant=None, with_asg=False, asz=None,
                 ss_extra=0, ps_extra=0, slot=None, ballot=None, n_planes=None):
        self.d, self.T, self.data_len, self.n, self.pop = d, T, data_len, n, pop
        self.kind, self.with_asg = kind, with_asg
        self.variant = (1 if kind == WAL else 2) if variant is None else variant
        self.asz = T if asz is None else asz
        self.L = -(-data_len // d)
        self.ss = round_up(self.L, 16) + ss_extra
        self.ps = n * self.ss + ps_extra
        n_planes = T if n_planes is None else n_planes                        # the fast path is handed one plane
        self.flat = rng.integers(0, 256, n_planes * self.ps, dtype=np.uint8)
        self.planes = np.lib.stride_tricks.as_strided(self.flat, shape=(n_planes, n, self.ss), strides=(self.ps, self.ss, 1))
        self.planes[:, :, self.L:round_up(self.L, 16)] = 0
        self.policies = np.ascontiguousarray(np.array(policies, dtype=np.uint64).astype(np.uint32)).reshape(-1, pop)
        self.pidx = None if pidx is None else np.ascontiguousarray(pidx, dtype=np.uint8)
        if slot is None:
            slot, ballot = _slots_ballots(rng, n)
        self.slot, self.ballot = np.ascontiguousarray(slot, dtype=np.uint64), np.ascontiguousarray(ballot, dtype=np.uint64)
        self._dev = None

    def row(self, g):
        k = 0 if self.pidx is None else int(self.pidx[g])
        return self.policies[k if k < len(self.policies) else 0]          # an index past the table selects policy 0

    def mask(self, g, peer):
        return int(self.row(g)[peer]) & ((1 << self.T) - 1)               # bits at or above T name no shard

    def want(self, wire, g, peer, mask=None):
        m = self.mask(g, peer) if mask is None else mask
        base = self.flat.ctypes.data + g * self.ss
        ptrs = [base + j * self.ps if (m >> j) & 1 else 0 for j in range(self.T)]
        return wire.encode(self.kind, self.variant, int(self.slot[g]), int(self.ballot[g]), self.d, self.T - self.d, self.data_len,
                           self.L, ptrs, self.row(g) if self.with_asg else None, self.asz)

    def spec(self, **over):
        f = dict(kind=self.kind, msg_variant=self.variant, data_shards=self.d, parity_shards=self.T - self.d, data_len=self.data_len,
                 population=self.pop, with_assignment=1 if self.with_asg else 0, assign_size=self.asz)
        f.update(over)
        return _lib.FrameSpec(**f)

    def dev(self):
        if self._dev is None:
            self._dev = dict(planes=_t(self.flat), pol=_t(self.policies), pidx=None if self.pidx is None else _t(self.pidx),
                             slot=_t(self.slot), ballot=_t(self.ballot))
        return self._dev


def _outputs(n, nbytes):
    return (torch.full((nbytes,), PAT, dtype=torch.uint8, device=DEV), torch.full((n,), OFF_PAT, dtype=torch.int64, device=DEV),
            torch.full((n,), LEN_PAT, dtype=torch.int32, device=DEV))


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _max_len(ctx, b, max_shards):
    return int(ctx.lib.ss_frame_accept_max_len(C.byref(b.spec()), max_shards))


def _pack(ctx, b, peer, stride, over=None):
    """ss_frame_accept_pack_dev called raw; `over` replaces arguments by name.  -> (rc, out, frame_off, frame_len)"""
    dv = b.dev()
    out, off, ln = _outputs(b.n, b.n * stride)
    a = dict(ctx=ctx.h, spec=b.spec(), planes=_ptr(dv["planes"]), ps=b.ps, ss=b.ss, pol=_ptr(dv["pol"]), npol=len(b.policies),
             pidx=_ptr(dv["pidx"]), peer=peer, slot=_ptr(dv["slot"]), ballot=_ptr(dv["ballot"]), n=b.n, out=_ptr(out), stride=stride,
             off=_ptr(off), ln=_ptr(ln))
    for k, v in (over or {}).items():
        a[k] = a[k] + v[1] if isinstance(v, tuple) and v[0] == "+" else v
    rc = ctx.lib.ss_frame_accept_pack_dev(a["ctx"], None if a["spec"] is None else C.byref(a["spec"]), a["planes"], a["ps"], a["ss"], a["pol"],
                                          a["npol"], a["pidx"], a["peer"], a["slot"], a["ballot"], a["n"], a["out"], a["stride"], a["off"], a["ln"])
    return rc, out, off, ln


def _fast(ctx, b, shard_idx, stride, over=None):
    """ss_frame_accept_batch_dev on plane `shard_idx` of the batch, raw"""
    dv = b.dev()
    out, off, ln = _outputs(b.n, b.n * stride)
    a = dict(ctx=ctx.h, plane=_ptr(dv["planes"]) + shard_idx * b.ps, ss=b.ss, idx=shard_idx, d=b.d, p=b.T - b.d, data_len=b.data_len,
             variant=b.variant, slot=_ptr(dv["slot"]), ballot=_ptr(dv["ballot"]), n=b.n, out=_ptr(out), stride=stride, off=_ptr(off), ln=_ptr(ln))
    for k, v in (over or {}).items():
        a[k] = a[k] + v[1] if isinstance(v, tuple) and v[0] == "+" else v
    rc = ctx.lib.ss_frame_accept_batch_dev(a["ctx"], a["plane"], a["ss"], a["idx"], a["d"], a["p"], a["data_len"], a["variant"], a["slot"],
                                           a["ballot"], a["n"], a["out"], a["stride"], a["off"], a["ln"])
    return rc, out, off, ln


def _ragged(ctx, b, peer, capacity, lens=None, shard_off=None, total=True, over=None):
    """ss_frame_accept_pack_ragged_dev raw, on the batch's planes as a ragged store: shard_off[g] = g * shard_stride"""
    dv = b.dev()
    out, off, ln = _outputs(b.n, capacity)
    lens_t = _t(np.full(b.n, b.data_len, dtype=np.uint32) if lens is None else lens)
    so_t = _t((np.arange(b.n, dtype=np.uint64) * np.uint64(b.ss)) if shard_off is None else shard_off)
    tot = torch.full((1,), OFF_PAT, dtype=torch.int64, device=DEV) if total else None
    a = dict(ctx=ctx.h, spec=b.spec(data_len=0), planes=_ptr(dv["planes"]), ps=b.ps, so=_ptr(so_t), lens=_ptr(lens_t), pol=_ptr(dv["pol"]),
             npol=len(b.policies), pidx=_ptr(dv["pidx"]), peer=peer, slot=_ptr(dv["slot"]), ballot=_ptr(dv["ballot"]), n=b.n, out=_ptr(out),
             cap=capacity, off=_ptr(off), ln=_ptr(ln), total=_ptr(tot))
    for k, v in (over or {}).items():
        a[k] = a[k] + v[1] if isinstance(v, tuple) and v[0] == "+" else v
    rc = ctx.lib.ss_frame_accept_pack_ragged_dev(a["ctx"], None if a["spec"] is None else C.byref(a["spec"]), a["planes"], a["ps"], a["so"],
                                                 a["lens"], a["pol"], a["npol"], a["pidx"], a["peer"], a["slot"], a["ballot"], a["n"], a["out"],
                                                 a["cap"], a["off"], a["ln"], a["total"])
    return rc, out, off, ln, tot


def _host(out, off, ln):
    return out.cpu().numpy(), off.cpu().numpy().view(np.uint64), ln.cpu().numpy().view(np.uint32)


def _untouched(out, off, ln):
    out, off, ln = _host(out, off, ln)
    return (out == PAT).all() and (off.view(np.int64) == OFF_PAT).all() and (ln == LEN_PAT).all()


def _check_frame(wire, b, g, got, want, mask):
    """byte-exact against the oracle's encoder, and the oracle's decoder reads back what went in.  -> the decoded frame"""
    assert got == want, (g, int(b.slot[g]), int(b.ballot[g]), hex(mask))
    dec = wire.decode(got, b.kind, b.with_asg)
    assert dec is not None and dec["length"] == len(got), g
    assert (dec["variant"], dec["slot"], dec["ballot"], dec["d"], dec["p"], dec["data_len"], dec["shard_len"]) == \
        (b.variant, int(b.slot[g]), int(b.ballot[g]), b.d, b.T - b.d, b.data_len, b.L), g
    assert [j for j in range(b.T) if dec["at"][j]] == [j for j in range(b.T) if (mask >> j) & 1], g
    for j in range(b.T):
        if dec["at"][j]:
            assert got[dec["at"][j]:dec["at"][j] + b.L] == b.planes[j, g, :b.L].tobytes(), (g, j)
    if b.with_asg:
        assert dec["assignment"] == [int(x) for x in b.row(g)] and dec["assign_size"] == b.asz, g
    return dec


def _check_uniform(wire, b, out, off, ln, stride, masks, fits=None, sample=None):
    """frames of a uniform packer: frame g inside slot g, placed so that its first carried shard's bytes are 16-byte
    aligned, every other byte of the buffer untouched.  masks[g]: the shards frame g carries; fits[g] False: the frame
    must not have been written.  sample: the frames compared byte for byte (all by default; frame_off / frame_len and
    the untouched bytes are checked for every frame either way).  -> frames written"""
    out, off, ln = _host(out, off, ln)
    n = b.n
    base = np.arange(n, dtype=np.uint64) * np.uint64(stride)
    rel = (off - base).astype(np.int64)
    assert (off >= base).all() and (rel < 16).all() and (rel + ln <= stride).all()
    cols = np.arange(stride, dtype=np.int64)[None, :]
    inside = (cols >= rel[:, None]) & (cols < (rel + ln.astype(np.int64))[:, None])
    assert (out.reshape(n, stride)[~inside] == PAT).all(), "a byte outside the frames was written"
    frames = {}
    for g in (range(n) if sample is None else sample):
        if fits is not None and not fits[g]:
            assert ln[g] == 0 and rel[g] == 0, g
            continue
        want = b.want(wire, g, None, masks[g])
        got = out[int(off[g]):int(off[g]) + int(ln[g])].tobytes()
        dec = _check_frame(wire, b, g, got, want, masks[g])
        if masks[g]:
            first = dec["at"][(masks[g] & -masks[g]).bit_length() - 1]
            assert rel[g] == -first % 16, (g, "the first carried shard is not 16-byte aligned in its slot")
        frames[g] = got
    return frames


# ---------------------------------------------------------------------------------------------
# 1-3: the length bounds, without a device
# ---------------------------------------------------------------------------------------------
def test_helpers_agree_with_the_oracle(oracle, wire):
    """what this file adds to the oracle is pinned to it: varint widths, and a WAL record as the peer frame's body less
    the PeerMessage tag"""
    for v in SPECIAL + VARIANTS + [249, 253, 254, 255, 256, (1 << 16) - 1, (1 << 32) + 1]:
        assert int(_vlen(v)) == len(oracle.varint(v)), v
    rng = np.random.default_rng(1)
    for d, p, dlen in ((3, 2, 10), (1, 0, 1), (5, 27, 70000 * 5), (16, 16, 251 * 16)):
        L = -(-dlen // d)
        sh = [rng.integers(0, 256, L, dtype=np.uint8) for _ in range(d + p)]
        for m in (1, 1 << (d + p - 1), (1 << (d + p)) - 1, 0b101 & ((1 << (d + p)) - 1)):
            for slot, ballot in ((0, 0), (251, 65536), (U64MAX, 1 << 32)):
                shards = [sh[j].tobytes() if (m >> j) & 1 else None for j in range(d + p)]
                ptrs = [sh[j].ctypes.data if (m >> j) & 1 else 0 for j in range(d + p)]
                assert wire.encode(PEER, 2, slot, ballot, d, p, dlen, L, ptrs) == oracle.frame_accept(2, slot, ballot, d, p, dlen, shards)
                assert wire.encode(WAL, 1, slot, ballot, d, p, dlen, L, ptrs) == oracle.wal_accept_data(slot, ballot, d, p, dlen, shards)
                fr = oracle.frame_accept(1, slot, ballot, d, p, dlen, shards)
                assert (len(fr) - 9).to_bytes(8, "big") + fr[9:] == oracle.wal_accept_data(slot, ballot, d, p, dlen, shards)


BOUND_DT = [(d, T) for T in (1, 2, 3, 5, 8, 16, 31, 32) for d in (1, 2, 3, 5, 8, 16, 31, 32) if d <= T]
BOUND_L = [1, 250, 251, 65535, 65536]


def _longest_frames(wire, kind, d, T, L, pop, asz, max_shards, zeros):
    """the longest frames a spec allows: widest variant, slot, ballot and policy rows, max_shards shards carried (the
    lowest and the highest indices)"""
    sets = {(1 << max_shards) - 1, ((1 << max_shards) - 1) << (T - max_shards)}
    for m in sorted(sets):
        ptrs = [zeros.ctypes.data if (m >> j) & 1 else 0 for j in range(T)]
        yield wire.encode(kind, U32MAX, U64MAX, U64MAX, d, T - d, L * d, L, ptrs, None if asz is None else [U32MAX] * pop, asz or 0)


@pytest.mark.parametrize("kind", [PEER, WAL])
@pytest.mark.parametrize("with_assignment", [0, 1])
def test_frame_accept_max_len_is_a_true_bound(wire, kind, with_assignment):
    """ss_frame_accept_max_len(spec, m) >= 15 bytes of alignment pad + the longest frame of that spec with m shards, for
    every code, population, assignment size and shard-length varint width; and the formula summerset_b200.api sizes the
    ragged packer's output with is the same number"""
    lib = _lib.load()
    assert lib.ss_frame_accept_max_len(None, 0) == 0 and lib.ss_frame_accept_max_len(None, 32) == 0
    zeros = np.zeros(65536, dtype=np.uint8)
    tight = 1 << 30
    for d, T in BOUND_DT:
        for pop, asz in ([(p, a) for p in (1, 2, 5, 12, 31, 32) for a in sorted({1, T, 63, 64})] if with_assignment else [(5, None)]):
            for L in BOUND_L:
                spec = _lib.FrameSpec(kind, U32MAX, d, T - d, L * d, pop, with_assignment, asz or 0)
                for ms in (0, 1, T):
                    bound = int(lib.ss_frame_accept_max_len(C.byref(spec), ms))
                    assert bound % 16 == 0
                    for fr in _longest_frames(wire, kind, d, T, L, pop, asz, ms, zeros):
                        assert len(fr) + 15 <= bound, (kind, d, T, L, pop, asz, ms, len(fr), bound)
                        tight = min(tight, bound - len(fr) - 15)
                assert int(frame_accept_room(L, T, pop, bool(with_assignment))) == int(lib.ss_frame_accept_max_len(C.byref(spec), T))
                Ls = np.array([L, 1, L + 1], dtype=np.int64)
                assert [int(x) for x in frame_accept_room(Ls, T, pop, bool(with_assignment))] == \
                    [int(lib.ss_frame_accept_max_len(C.byref(_lib.FrameSpec(kind, 2, d, T - d, int(x) * d, pop, with_assignment, asz or 0)), T)) for x in Ls]
    assert tight < 32                                       # the bound is a bound, not a guess with a page to spare


def test_fast_path_stride_bound_holds_the_widest_frame(wire):
    """ss_frame_accept_batch_dev documents frame_stride >= shard_len + 96 + d + p: room for 15 bytes of pad and the widest
    single-shard frame"""
    zeros = np.zeros(65537, dtype=np.uint8)
    for d, T in ((1, 1), (3, 5), (1, 5), (5, 5), (125, 250), (249, 250), (1, 250)):
        for L in L_EDGES:
            for idx in sorted({0, T // 2, T - 1}):
                ptrs = [zeros.ctypes.data if j == idx else 0 for j in range(T)]
                fr = wire.encode(PEER, U32MAX, U64MAX, U64MAX, d, T - d, L * d, L, ptrs)
                assert len(fr) + 15 <= L + 96 + T, (d, T, L, idx, len(fr))


# ---------------------------------------------------------------------------------------------
# 4: general packer, code x population x peer x kind
# ---------------------------------------------------------------------------------------------
CODES = [(1, 1), (1, 2), (2, 3), (3, 5), (4, 7), (5, 9), (6, 10), (8, 16), (13, 24), (16, 32), (32, 32), (31, 32)]
POPULATIONS = [1, 2, 3, 5, 7, 12, 16, 32]


def _peers(pop):
    return sorted({0, pop // 2, pop - 1})


def _policy_table(oracle, rng, d, T, pop):
    """every shape of policy row: RSPaxos's one shard per replica, Crossword's balanced assignments, unbalanced rows, a
    replica given nothing, every bit set, bits at and above T"""
    full = (1 << T) - 1
    tabs = [[1 << (r % T) for r in range(pop)]]
    tabs += [[int(x) for x in oracle.cw_brr_assignment(pop, T, spr)] for spr in sorted({1, max(1, T // pop), d, T})]
    tabs += [[int(x) for x in rng.integers(0, full + 1, pop)] for _ in range(2)]
    for peer in _peers(pop):
        row = [int(x) for x in rng.integers(0, full + 1, pop)]
        row[peer] = 0
        tabs.append(row)
    tabs.append([full] * pop)
    tabs.append([int(x) for x in rng.integers(0, 1 << 32, pop)])          # bits at and above T: dropped from the shards carried,
    tabs.append([U32MAX] * pop)                                           # kept in the assignment bitmaps
    tabs.append([(1 << 31) | int(x) for x in rng.integers(0, full + 1, pop)])
    return tabs


@pytest.mark.gpu
@pytest.mark.parametrize("pop", POPULATIONS)
@pytest.mark.parametrize("d,T", CODES)
def test_general_packer_code_population_matrix(ctx, oracle, wire, d, T, pop):
    rng = np.random.default_rng(1000 * T + 32 * d + pop)
    n = 300
    tabs = _policy_table(oracle, rng, d, T, pop)
    pidx = rng.integers(0, len(tabs), n).astype(np.uint8)
    pidx[rng.random(n) < 0.05] = rng.integers(len(tabs), 256)            # out of range: policy 0
    pidx[:4] = [len(tabs), 255, 0, len(tabs) - 1]
    for name, (kind, with_asg) in KINDS.items():
        b = _Batch(rng, d, T, int(rng.integers(1, 40 * d + 1)), n, pop, tabs, pidx, kind=kind, with_asg=with_asg)
        stride = _max_len(ctx, b, T)
        for peer in _peers(pop):
            rc, out, off, ln = _pack(ctx, b, peer, stride)
            assert rc == 0 and ctx.device_status() == 0, (name, peer)
            _check_uniform(wire, b, out, off, ln, stride, [b.mask(g, peer) for g in range(n)])
    # policy_idx == NULL: every codeword takes policy 0
    b = _Batch(rng, d, T, int(rng.integers(1, 40 * d + 1)), n, pop, tabs[3:] + tabs[:3], None, with_asg=True)
    peer = _peers(pop)[-1]
    rc, out, off, ln = _pack(ctx, b, peer, _max_len(ctx, b, T))
    assert rc == 0 and ctx.device_status() == 0
    _check_uniform(wire, b, out, off, ln, _max_len(ctx, b, T), [int(b.policies[0][peer]) & ((1 << T) - 1)] * n)


# ---------------------------------------------------------------------------------------------
# 5: shard lengths and strides
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("L", L_EDGES)
@pytest.mark.parametrize("d,T", [(3, 5), (16, 32), (1, 32)])
def test_general_packer_shard_length_and_stride_edges(ctx, wire, d, T, L):
    """the Some length prefix changes width at L = 251 and 65536 and moves every later byte; the second and later shards
    of a frame start at (L + prefix) mod 16 past an aligned address, so 1, 2 and T shards per frame over these lengths put
    shard copies on every destination alignment; slots and planes wider than the shards must not leak into the frames"""
    rng = np.random.default_rng(77 * L + T + d)
    pop = 5
    n = 24 if L <= 4097 else 5
    full = (1 << T) - 1
    tabs = [[1 << (r % T) for r in range(pop)], [0b11 << (r % (T - 1)) for r in range(pop)], [full] * pop,
            [(1 | 1 << (T - 1)) for _ in range(pop)]]
    pidx = (np.arange(n) % len(tabs)).astype(np.uint8)
    for data_len in sorted({L * d, (L - 1) * d + 1}):
        for k, (ss_extra, ps_extra) in enumerate(((0, 0), (16, 16), (4096, 65536))):
            kind, with_asg = list(KINDS.values())[(k + L) % 3]
            b = _Batch(rng, d, T, data_len, n, pop, tabs, pidx, kind=kind, with_asg=with_asg, ss_extra=ss_extra, ps_extra=ps_extra)
            assert b.L == L
            stride = _max_len(ctx, b, T)
            peer = (k + L) % pop
            rc, out, off, ln = _pack(ctx, b, peer, stride)
            assert rc == 0 and ctx.device_status() == 0
            _check_uniform(wire, b, out, off, ln, stride, [b.mask(g, peer) for g in range(n)])


# ---------------------------------------------------------------------------------------------
# 6: varint widths
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kind", list(KINDS))
def test_general_packer_varint_widths(ctx, wire, kind, variant):
    """msg_variant of every width with every pair of slot and ballot widths; assignment bitmaps of 1, 5, 63 and 64 bits
    (also narrower than the code) holding rows at 250 / 251 / 65535 / 65536 / 2^31"""
    rng = np.random.default_rng(variant % 1000 + len(kind))
    k, with_asg = KINDS[kind]
    rows = [250, 251, 65535, 65536, 1 << 31, (1 << 31) | 251, 0, 7, U32MAX]
    for (d, T), pop in (((3, 5), 5), ((16, 32), 9), ((5, 8), 3)):
        tabs = [[rows[(r + s) % len(rows)] for r in range(pop)] for s in range(len(rows))]
        n = 121
        pidx = rng.integers(0, len(tabs), n).astype(np.uint8)
        for asz in ((1, 5, 63, 64) if with_asg else (T,)):
            b = _Batch(rng, d, T, int(rng.integers(1, 100 * d)), n, pop, tabs, pidx, kind=k, variant=variant, with_asg=with_asg, asz=asz)
            stride = _max_len(ctx, b, T)
            peer = int(rng.integers(0, pop))
            rc, out, off, ln = _pack(ctx, b, peer, stride)
            assert rc == 0 and ctx.device_status() == 0
            _check_uniform(wire, b, out, off, ln, stride, [b.mask(g, peer) for g in range(n)])


# ---------------------------------------------------------------------------------------------
# 7: frames that fit beside frames that do not
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_general_packer_fit_is_decided_frame_by_frame(ctx, wire):
    """header widths differ per frame (slot / ballot varints), so with a slot exact for the narrowest frames some fit and
    their neighbours do not; a frame that does not fit -- counting the pad that aligns its first shard -- leaves its whole
    slot untouched, frame_len 0, frame_off at the slot's start, and sets the overflow bit once"""
    rng = np.random.default_rng(7)
    d, T, pop, peer = 3, 5, 5, 1
    widths = np.array([3, 300, 70000, 1 << 33], dtype=np.uint64)             # 1, 3, 5 and 9 byte varints
    n = 64
    i = np.arange(n)
    pad_counts = 0
    for data_len in (1, 7, 20, 48, 100, 250 * 3, 251 * 3, 4000):
        b = _Batch(rng, d, T, data_len, n, pop, [[1 << r for r in range(pop)]], None, slot=widths[i % 4] + (i // 16).astype(np.uint64),
                   ballot=widths[i // 4 % 4])
        lens, pads = [], []
        for g in range(n):
            fr = b.want(wire, g, peer)
            lens.append(len(fr))
            pads.append(-wire.decode(fr, PEER, False)["at"][peer] % 16)
        lens, pads = np.array(lens), np.array(pads)
        stride = round_up(int(pads[0] + lens[0]), 16)                        # frame 0: one-byte slot and ballot
        fits = pads + lens <= stride
        assert fits[0] and not fits.all() and not fits[15] and lens.max() == lens[15] == lens[0] + 16
        pad_counts += int(((lens <= stride) & ~fits).sum())
        rc, out, off, ln = _pack(ctx, b, peer, stride)
        assert rc == 0
        assert ctx.device_status() == OVERFLOW and ctx.device_status() == 0  # read once, cleared
        written = _check_uniform(wire, b, out, off, ln, stride, [1 << peer] * n, fits=fits)
        assert sorted(written) == [g for g in range(n) if fits[g]]
        rc, out, off, ln = _pack(ctx, b, peer, stride + 16)
        assert rc == 0 and ctx.device_status() == 0
        assert len(_check_uniform(wire, b, out, off, ln, stride + 16, [1 << peer] * n)) == n
    assert pad_counts > 0          # some frame was refused for its pad alone


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [PEER, WAL])
def test_general_packer_fills_a_slot_of_exactly_max_len(ctx, wire, kind):
    """frame_stride == ss_frame_accept_max_len(spec, T) holds the spec's longest frames"""
    rng = np.random.default_rng(70 + kind)
    for (d, T), pop, L in (((3, 5), 5, 65536), ((16, 32), 32, 251), ((1, 1), 1, 1), ((31, 32), 12, 65535)):
        n = 3
        full = (1 << T) - 1
        b = _Batch(rng, d, T, L * d, n, pop, [[U32MAX] * pop], None, kind=kind, variant=U32MAX, with_asg=True, asz=64,
                   slot=np.full(n, U64MAX, dtype=np.uint64), ballot=np.array([U64MAX, U64MAX - 1, 1 << 32], dtype=np.uint64))
        stride = _max_len(ctx, b, T)
        rc, out, off, ln = _pack(ctx, b, pop - 1, stride)
        assert rc == 0 and ctx.device_status() == 0
        assert len(_check_uniform(wire, b, out, off, ln, stride, [full] * n)) == n


# ---------------------------------------------------------------------------------------------
# 8: past the grid cap
# ---------------------------------------------------------------------------------------------
def _sample(n, cap):
    s = np.concatenate([np.arange(64), np.arange(n - 64, n), np.arange(0, n, max(1, n // 4200)), np.arange(cap - 64, cap + 64),
                        np.arange(2 * cap - 64, 2 * cap + 37)])
    return [int(g) for g in np.unique(s[(s >= 0) & (s < n)])]


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["general", "fast"])
def test_packers_past_the_grid_cap_and_back_to_back(ctx, wire, path):
    """the launches are capped at sm_count * 64 CTAs of 8 warps, a warp per frame: more frames than that go round the
    grid-stride loop.  Two calls on different inputs are enqueued with nothing between them."""
    cap = ctx.sm_count * 512
    n = 2 * cap + 37
    d, T, pop, peer = 3, 5, 5, 2
    batches = [_Batch(np.random.default_rng(80 + k), d, T, dl, n, pop, [[1 << r for r in range(pop)]], None) for k, dl in enumerate((16, 5))]
    for b in batches:
        b.dev()
    stride = round_up(max(max(_max_len(ctx, b, 1), b.L + 96 + T) for b in batches), 16)
    torch.cuda.synchronize()
    launches = ctx.launches
    res = [(_pack(ctx, b, peer, stride) if path == "general" else _fast(ctx, b, peer, stride)) for b in batches]
    assert ctx.launches == launches + 2
    assert ctx.device_status() == 0
    for b, (rc, out, off, ln) in zip(batches, res):
        assert rc == 0
        base = len(b.want(wire, 0, peer)) - int(_vlen(b.slot[0])) - int(_vlen(b.ballot[0]))
        assert (ln.cpu().numpy().view(np.uint32) == base + _vlen(b.slot) + _vlen(b.ballot)).all()
        assert len(_check_uniform(wire, b, out, off, ln, stride, [1 << peer] * n, sample=_sample(n, cap))) >= 4096


# ---------------------------------------------------------------------------------------------
# 9: the single-shard fast path
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("d,p", [(1, 0), (1, 1), (3, 2), (8, 8), (16, 16), (125, 125), (249, 1)])
def test_fast_path_matrix(ctx, wire, d, p):
    """codes up to the documented T = 250, the shard first, last and beyond a warp's width of None tags on either side,
    every shard-length edge, every msg_variant width, frame_stride exactly round_up(L + 96 + d + p, 16) and wider, shard
    slots wider than the padded shard; the shard's bytes 16-byte aligned in every frame"""
    rng = np.random.default_rng(900 + d + p)
    T = d + p
    n = 23
    i = np.arange(n)
    sp = np.array(SPECIAL, dtype=np.uint64)
    cell = 0
    for idx in sorted({j for j in (0, 1, 31, 32, 33, T - 34, T - 1) if 0 <= j < T}):
        for L in L_EDGES:
            cell += 1
            data_len = L * d if cell % 2 else (L - 1) * d + 1
            b = _Batch(rng, d, T, data_len, n, 1, [[0]], None, variant=VARIANTS[cell % len(VARIANTS)], ss_extra=(0, 16, 4096)[cell % 3],
                       slot=sp[(i + cell) % 11], ballot=sp[(i * 3 + cell // 11) % 11], n_planes=1)
            stride = round_up(L + 96 + T, 16) + (0, 48)[cell // 3 % 2]
            rc, out, off, ln = _fast(ctx, b, 0, stride, dict(idx=idx))
            assert rc == 0 and ctx.device_status() == 0, (idx, L)
            # the batch's only plane is handed over as shard idx: the oracle is given the same bytes under that index
            out_h, off_h, ln_h = _host(out, off, ln)
            base = np.arange(n, dtype=np.uint64) * np.uint64(stride)
            rel = (off_h - base).astype(np.int64)
            assert (off_h >= base).all() and (rel < 16).all() and (rel + ln_h <= stride).all()
            cols = np.arange(stride, dtype=np.int64)[None, :]
            inside = (cols >= rel[:, None]) & (cols < (rel + ln_h.astype(np.int64))[:, None])
            assert (out_h.reshape(n, stride)[~inside] == PAT).all()
            for g in range(n):
                ptrs = [b.flat.ctypes.data + g * b.ss if j == idx else 0 for j in range(T)]
                want = wire.encode(PEER, b.variant, int(b.slot[g]), int(b.ballot[g]), d, p, data_len, L, ptrs)
                got = out_h[int(off_h[g]):int(off_h[g]) + int(ln_h[g])].tobytes()
                assert got == want, (idx, L, g)
                dec = wire.decode(got, PEER, False)
                assert dec and (dec["variant"], dec["slot"], dec["ballot"], dec["d"], dec["p"], dec["data_len"], dec["shard_len"]) == \
                    (b.variant, int(b.slot[g]), int(b.ballot[g]), d, p, data_len, L)
                assert [j for j in range(T) if dec["at"][j]] == [idx]
                assert got[dec["at"][idx]:dec["at"][idx] + L] == b.planes[0, g, :L].tobytes()
                assert (int(off_h[g]) + dec["at"][idx]) % 16 == 0


# ---------------------------------------------------------------------------------------------
# 10: the three packers against each other
# ---------------------------------------------------------------------------------------------
def _check_ragged(wire, b, out, off, ln, tot, masks, lens=None, written=None):
    """the packed layout: frame g's region is round_up(pad + len, 16) bytes, the regions follow each other in group
    order, frame_off[g] = region start + pad; nothing outside the frames is written, nor past the total.  -> frames"""
    out, off, ln = _host(out, off, ln)
    at, frames, covered = 0, {}, np.zeros(out.size, dtype=bool)
    for g in range(b.n):
        if written is not None and not written[g]:
            assert ln[g] == 0, g
            continue
        if lens is not None:
            b.data_len, b.L = int(lens[g]), -(-int(lens[g]) // b.d)
        want = b.want(wire, g, None, masks[g])
        got = out[int(off[g]):int(off[g]) + int(ln[g])].tobytes()
        dec = _check_frame(wire, b, g, got, want, masks[g])
        pad = int(off[g]) - at
        assert 0 <= pad < 16, g
        if masks[g]:
            assert pad == -dec["at"][(masks[g] & -masks[g]).bit_length() - 1] % 16, g
        covered[int(off[g]):int(off[g]) + len(got)] = True
        at += round_up(pad + len(got), 16)
        frames[g] = got
    assert (out[~covered] == PAT).all()
    if tot is not None:
        assert int(tot.cpu()[0]) == at
    return frames, at


@pytest.mark.gpu
@pytest.mark.parametrize("d,T,pop", [(3, 5, 5), (4, 7, 7), (8, 16, 16), (1, 3, 3), (16, 32, 32)])
def test_three_packers_agree_on_single_shard_frames(ctx, wire, d, T, pop):
    rng = np.random.default_rng(100 + T)
    n = 150
    for data_len in (1, 251 * d, int(rng.integers(2, 3000))):
        b = _Batch(rng, d, T, data_len, n, pop, [[1 << (r % T) for r in range(pop)]], None)
        stride = round_up(max(_max_len(ctx, b, 1), b.L + 96 + T), 16)
        for peer in _peers(pop):
            masks = [1 << peer] * n
            rc, out, off, ln = _pack(ctx, b, peer, stride)
            assert rc == 0
            general = _check_uniform(wire, b, out, off, ln, stride, masks)
            rc, out2, off2, ln2 = _fast(ctx, b, peer, stride)
            assert rc == 0
            assert torch.equal(out, out2) and torch.equal(off, off2) and torch.equal(ln, ln2)
            rc, out3, off3, ln3, tot = _ragged(ctx, b, peer, n * stride)
            assert rc == 0 and ctx.device_status() == 0
            sent = b.slot != U64MAX                                          # the ragged packer frames no such codeword
            ragged, _ = _check_ragged(wire, b, out3, off3, ln3, tot, masks, written=sent)
            assert ragged == {g: general[g] for g in range(n) if sent[g]}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
def test_general_and_ragged_packers_agree_on_multi_shard_frames(ctx, oracle, wire, kind):
    k, with_asg = KINDS[kind]
    for d, T, pop in ((3, 5, 5), (5, 10, 5), (16, 32, 8)):
        rng = np.random.default_rng(110 + T + len(kind))
        n = 120
        tabs = _policy_table(oracle, rng, d, T, pop)
        pidx = rng.integers(0, len(tabs) + 2, n).astype(np.uint8)
        b = _Batch(rng, d, T, int(rng.integers(1, 2000)), n, pop, tabs, pidx, kind=k, with_asg=with_asg)
        stride = _max_len(ctx, b, T)
        for peer in _peers(pop):
            masks = [b.mask(g, peer) for g in range(n)]
            rc, out, off, ln = _pack(ctx, b, peer, stride)
            assert rc == 0
            general = _check_uniform(wire, b, out, off, ln, stride, masks)
            rc, out3, off3, ln3, tot = _ragged(ctx, b, peer, n * stride)
            assert rc == 0 and ctx.device_status() == 0
            sent = b.slot != U64MAX
            ragged, _ = _check_ragged(wire, b, out3, off3, ln3, tot, masks, written=sent)
            assert ragged == {g: general[g] for g in range(n) if sent[g]}


@pytest.mark.gpu
def test_ragged_packer_called_raw(ctx, oracle, wire):
    """what summerset_b200.api pins: assign_size other than T, total == NULL, a plane_stride wider than the store; lengths
    that differ per codeword, codewords that are skipped (length 0, slot UINT64_MAX), and a capacity that ends mid-batch"""
    rng = np.random.default_rng(120)
    d, T, pop, n, peer = 3, 5, 5, 200, 3
    tabs = _policy_table(oracle, rng, d, T, pop)
    pidx = rng.integers(0, len(tabs), n).astype(np.uint8)
    top = 251 * d
    b = _Batch(rng, d, T, top, n, pop, tabs, pidx, with_asg=True, asz=64, ps_extra=65536 + 16)
    lens = rng.integers(1, top + 1, n).astype(np.uint32)
    lens[:8] = [1, d, d + 1, 250 * d, 250 * d + 1, top, 0, 16]
    lens[rng.random(n) < 0.05] = 0
    b.slot[5::17] = U64MAX
    b._dev = None
    written = (lens != 0) & (b.slot != U64MAX)
    # slots of the store hold a codeword's shard in their first ceil(len / d) bytes: shorter codewords read a prefix
    masks = [b.mask(g, peer) for g in range(n)]
    cap = n * _max_len(ctx, b, T)
    rc, out, off, ln, tot = _ragged(ctx, b, peer, cap, lens=lens)
    assert rc == 0 and ctx.device_status() == 0
    _, total = _check_ragged(wire, b, out, off, ln, tot, masks, lens=lens, written=written)
    rc, out2, off2, ln2, _ = _ragged(ctx, b, peer, cap, lens=lens, total=False)
    assert rc == 0 and ctx.device_status() == 0
    assert torch.equal(out, out2) and torch.equal(ln, ln2)
    # a capacity that ends inside the batch: the frames whose regions end at or before it are written, the rest are not
    off_h, ln_h = off.cpu().numpy().view(np.uint64), ln.cpu().numpy().view(np.uint32)
    ends = np.array([round_up(int(off_h[g]) + int(ln_h[g]), 16) if written[g] else 0 for g in range(n)])
    cut = int(np.sort(ends[ends > 0])[len(ends[ends > 0]) // 2])
    rc, out3, off3, ln3, tot3 = _ragged(ctx, b, peer, cut, lens=lens)
    assert rc == 0 and ctx.device_status() == OVERFLOW and ctx.device_status() == 0
    assert int(tot3.cpu()[0]) == total
    fit = written & (ends <= cut)
    assert fit.any() and not fit[written].all()
    ln3_h = ln3.cpu().numpy().view(np.uint32)
    assert (ln3_h[fit] == ln_h[fit]).all() and (ln3_h[~fit] == 0).all()
    assert (off3.cpu().numpy().view(np.uint64)[fit] == off_h[fit]).all()
    assert (out3.cpu().numpy() == out.cpu().numpy()[:cut]).all()           # a region ends at the cut: the same bytes before it


# ---------------------------------------------------------------------------------------------
# 11: refusals
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_packers_refuse_what_the_abi_excludes(ctx, oracle, wire):
    """every refusal is SS_ERR_INVALID_ARG, launches nothing and writes nothing; the next valid call succeeds"""
    rng = np.random.default_rng(11)
    d, T, pop, n, peer = 3, 5, 5, 40, 2
    b = _Batch(rng, d, T, 100 * d, n, pop, [[1 << r for r in range(pop)], [0b111] * pop], (np.arange(n) % 2).astype(np.uint8), with_asg=True)
    stride = round_up(max(_max_len(ctx, b, T), b.L + 96 + T), 16)
    plus8 = ("+", 8)
    general = [dict(spec=b.spec(data_shards=0)), dict(spec=b.spec(data_shards=3, parity_shards=30)), dict(spec=b.spec(data_shards=33, parity_shards=0)),
               dict(spec=b.spec(data_len=0)), dict(spec=b.spec(kind=2)), dict(spec=b.spec(kind=U32MAX)), dict(spec=b.spec(population=0)),
               dict(spec=b.spec(population=33)), dict(peer=pop), dict(peer=U32MAX), dict(npol=0), dict(spec=b.spec(assign_size=0)),
               dict(spec=b.spec(assign_size=65)), dict(stride=plus8), dict(out=plus8), dict(planes=plus8), dict(ps=plus8), dict(ss=plus8),
               dict(ss=round_up(b.L, 16) - 16), dict(planes=0), dict(pol=0), dict(slot=0), dict(ballot=0), dict(out=0), dict(off=0), dict(ln=0),
               dict(ctx=None), dict(spec=None)]
    fast = [dict(d=0), dict(d=126, p=125), dict(d=250, p=1), dict(idx=T), dict(idx=U32MAX), dict(data_len=0), dict(stride=plus8), dict(out=plus8),
            dict(plane=plus8), dict(ss=plus8), dict(stride=round_up(b.L + 96 + T, 16) - 16), dict(plane=0), dict(slot=0), dict(ballot=0),
            dict(out=0), dict(off=0), dict(ln=0), dict(ctx=None)]
    ragged = [dict(spec=b.spec(data_shards=0)), dict(spec=b.spec(data_shards=3, parity_shards=30)), dict(spec=b.spec(kind=2)),
              dict(spec=b.spec(population=0)), dict(spec=b.spec(population=33)), dict(peer=pop), dict(npol=0), dict(spec=b.spec(assign_size=0)),
              dict(spec=b.spec(assign_size=65)), dict(out=plus8), dict(planes=plus8), dict(ps=plus8), dict(planes=0), dict(so=0), dict(lens=0),
              dict(pol=0), dict(slot=0), dict(ballot=0), dict(out=0), dict(off=0), dict(ln=0), dict(ctx=None), dict(spec=None)]
    torch.cuda.synchronize()
    launches = ctx.launches
    for over in general:
        rc, out, off, ln = _pack(ctx, b, peer, stride, over)
        assert rc == INVALID, over
        assert _untouched(out, off, ln), over
    for over in fast:
        rc, out, off, ln = _fast(ctx, b, peer, stride, over)
        assert rc == INVALID, over
        assert _untouched(out, off, ln), over
    for over in ragged:
        rc, out, off, ln, tot = _ragged(ctx, b, peer, n * stride, over=over)
        assert rc == INVALID, over
        assert _untouched(out, off, ln) and int(tot.cpu()[0]) == OFF_PAT, over
    # n == 0 succeeds with no buffer at all
    lib = ctx.lib
    assert lib.ss_frame_accept_pack_dev(ctx.h, C.byref(b.spec()), None, 0, 0, None, 0, None, 0, None, None, 0, None, 0, None, None) == 0
    assert lib.ss_frame_accept_batch_dev(ctx.h, None, 0, 0, 0, 0, 0, 0, None, None, 0, None, 0, None, None) == 0
    assert lib.ss_frame_accept_pack_ragged_dev(ctx.h, C.byref(b.spec()), None, 0, None, None, None, 0, None, 0, None, None, 0, None, 0, None,
                                               None, None) == 0
    assert ctx.launches == launches and ctx.device_status() == 0
    # assign_size is not looked at without an assignment
    masks = [b.mask(g, peer) for g in range(n)]
    for asz in (0, 65):
        plain = _Batch(np.random.default_rng(12), d, T, b.data_len, n, pop, b.policies, b.pidx, with_asg=False, asz=asz)
        rc, out, off, ln = _pack(ctx, plain, peer, stride)
        assert rc == 0 and ctx.device_status() == 0
        _check_uniform(wire, plain, out, off, ln, stride, masks)
        rc, out, off, ln, tot = _ragged(ctx, plain, peer, n * stride)
        assert rc == 0 and ctx.device_status() == 0
        _check_ragged(wire, plain, out, off, ln, tot, masks, written=plain.slot != U64MAX)
    # and the calls refused above go through unchanged
    rc, out, off, ln = _pack(ctx, b, peer, stride)
    assert rc == 0 and ctx.device_status() == 0
    _check_uniform(wire, b, out, off, ln, stride, masks)
    rc, out, off, ln = _fast(ctx, b, peer, stride)
    assert rc == 0 and ctx.device_status() == 0
    one = _Batch(np.random.default_rng(11), d, T, b.data_len, n, pop, [[1 << r for r in range(pop)]], None, variant=2)
    one.flat[:] = b.flat
    one.slot, one.ballot = b.slot, b.ballot
    _check_uniform(wire, one, out, off, ln, stride, [1 << peer] * n)
    rc, out, off, ln, tot = _ragged(ctx, b, peer, n * stride)
    assert rc == 0 and ctx.device_status() == 0
    _check_ragged(wire, b, out, off, ln, tot, masks, written=b.slot != U64MAX)
