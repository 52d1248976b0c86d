"""The bulk-copy RS(3,2) accept-step kernel (rs32_accept_bulk_kernel, selected by variant bit 18) against the row kernel
that runs the accept step by default and against the CPU oracle, bit-exact: parity planes with guard bands around
every buffer and in the slack of every shard slot, commit words and commit_bar with guards at both ends."""
import numpy as np
import pytest
import torch

from summerset_b200 import workloads as wl
from summerset_b200.api import SS_RS_OUT_PADDED16, ReedSolomon, round_up, shard_len
from summerset_b200._lib import check

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D, P, R, THRESH = 3, 2, 5, 4
BULK = 1 << 18
GUARD = 64                      # bytes (parity) / elements (commit words, commit_bar) of guard band on each side
SENT = 0xC3
# stage edges: one byte, one vector +-1, three vectors +-1, the cfg3 payload +-1, and the largest payload that still
# fits 256 columns (L = 4096)
LENS = [1, 15, 16, 17, 47, 48, 49, 4095, 4096, 4097, 12288]


def _step(ctx, rs, variant, data, data_len, stride, n, ss, tally, planes, with_bar):
    """One fused accept step (or plain encode when tally is False) into guarded buffers; returns host copies."""
    ps = n * ss
    par = torch.full((2 * GUARD + P * ps,), SENT, dtype=torch.uint8, device=DEV)
    com = torch.full((n + 2 * GUARD,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device=DEV)
    bar = torch.full((n + 2 * GUARD,), 0x3C3C3C3C, dtype=torch.int32, device=DEV)
    base = par.data_ptr() + GUARD
    assert base % 16 == 0
    rs.set_variant(variant)
    if tally:
        check(ctx.lib.ss_accept_step_fused_dev(rs.h, data.data_ptr(), stride, data_len, n, base, ps, ss, SS_RS_OUT_PADDED16,
                                               planes.data_ptr(), R, THRESH, com.data_ptr() + 8 * GUARD,
                                               bar.data_ptr() + 4 * GUARD if with_bar else None))
    else:
        check(ctx.lib.ss_rs_encode_uniform_dev(rs.h, data.data_ptr(), stride, data_len, n, base, ps, ss, SS_RS_OUT_PADDED16))
    torch.cuda.synchronize()
    kernel = rs.last_kernel()
    rs.set_variant(0)
    return par.cpu().numpy(), com.cpu().numpy().view(np.uint64), bar.cpu().numpy().view(np.uint32), kernel


def _check(ctx, oracle, data_len, n, stride_extra=0, ss_extra=0, tally=True, with_bar=True, seed=0, bulk=BULK):
    rs = ReedSolomon(ctx, D, P)
    stride = round_up(data_len, 16) + stride_extra
    L = shard_len(data_len, D)
    vb = round_up(L, 16)
    ss = vb + ss_extra
    data_np = wl.payload_uniform(n, data_len, stride=stride, seed_extra=seed + data_len)
    data = torch.from_numpy(data_np).to(DEV)
    planes_np = wl.cfg2_planes(n, R, 0.9, seed_extra=seed + n)
    planes = torch.from_numpy(planes_np.view(np.int64)).to(DEV)
    new = _step(ctx, rs, bulk, data, data_len, stride, n, ss, tally, planes, with_bar)
    old = _step(ctx, rs, 0, data, data_len, stride, n, ss, tally, planes, with_bar)
    assert new[3] == ("rs32_accept_bulk_kernel+tally" if tally else "rs32_accept_bulk_kernel")
    assert old[3].startswith("rs32_encode_row_kernel")
    # bit-exact against the row kernel: every byte of the parity buffer (guards included), commit words, commit_bar
    for i, what in enumerate(("parity buffer", "commit words", "commit_bar")):
        assert (new[i] == old[i]).all(), f"{what} differs from the row kernel"
    par = new[0]
    assert (par[:GUARD] == SENT).all() and (par[GUARD + P * n * ss:] == SENT).all(), "guard band around the planes written"
    body = par[GUARD:GUARD + P * n * ss].reshape(P, n, ss)
    assert (body[:, :, vb:] == SENT).all(), "bytes past vpc*16 in a shard slot written"
    want = oracle.rs_encode_uniform(D, P, data_np, data_len)
    assert (body[:, :, :vb] == want).all(), "parity differs from the oracle"
    com, bar = new[1], new[2]
    if tally:
        cw, bw = oracle.tally_planes(planes_np, THRESH)
        assert (com[GUARD:GUARD + n] == cw).all(), "commit words differ from the oracle"
        assert (com[:GUARD] == 0x5A5A5A5A5A5A5A5A).all() and (com[GUARD + n:] == 0x5A5A5A5A5A5A5A5A).all()
        if with_bar:
            assert (bar[GUARD:GUARD + n] == bw).all(), "commit_bar differs from the oracle"
    if not (tally and with_bar):
        assert (bar == 0x3C3C3C3C).all(), "commit_bar written without being asked for"
    if not tally:
        assert (com == 0x5A5A5A5A5A5A5A5A).all(), "commit words written by a plain encode"
    assert (bar[:GUARD] == 0x3C3C3C3C).all() and (bar[GUARD + n:] == 0x3C3C3C3C).all()


@pytest.mark.parametrize("data_len", LENS)
@pytest.mark.parametrize("n", [1, 7, 1531])
@pytest.mark.parametrize("mode", ["tally", "tally_no_bar", "encode_only"])
def test_bulk_matches_row_kernel_and_oracle(ctx, oracle, data_len, n, mode):
    """n = 1; fewer codewords than one CTA's ring of stages; a count that no CTA range divides"""
    _check(ctx, oracle, data_len, n, tally=mode != "encode_only", with_bar=mode == "tally")


@pytest.mark.parametrize("data_len", [17, 1000, 4096, 12288])
@pytest.mark.parametrize("stride_extra,ss_extra", [(16, 0), (0, 32), (48, 16), (4096, 0)])
def test_bulk_strides(ctx, oracle, data_len, stride_extra, ss_extra):
    """data_stride > round_up(len, 16) (slack bytes are non-zero and must be masked) and shard_stride > vpc*16
    (the slack of every shard slot stays untouched); 4999 codewords: the last CTA's range is shorter"""
    _check(ctx, oracle, data_len, 4999, stride_extra=stride_extra, ss_extra=ss_extra, seed=stride_extra + ss_extra)


@pytest.mark.parametrize("tuning", [1 << 19, 2 << 19, 3 << 19, 1 << 21, (3 << 19) | (1 << 21)])
def test_bulk_tuning_bits(ctx, oracle, tuning):
    """the tuning bits (resident CTAs per SM, interleaved codewords) change the schedule, never the bytes"""
    _check(ctx, oracle, 4096, 4999, stride_extra=16, ss_extra=16, bulk=BULK | tuning)


def test_bulk_cfg3_full_size(ctx, oracle):
    """the bench shape: 2^20 groups x 4096 B, 5 replicas, tally 4 of 5 -- every byte equal to the row kernel's,
    1024 sampled groups equal to the oracle"""
    n, data_len = 1 << 20, 4096
    rs = ReedSolomon(ctx, D, P)
    L, ds, ps = rs.parity_layout(data_len, n)
    gen = torch.Generator(device=DEV); gen.manual_seed(4242)
    data = torch.randint(0, 256, (n, data_len), dtype=torch.uint8, device=DEV, generator=gen)
    planes = torch.randint(0, 256, (R, n * 8), dtype=torch.uint8, device=DEV, generator=gen).view(torch.int64)
    res = {}
    for v in (BULK, 0):
        par = torch.full((P, n, ds), SENT, dtype=torch.uint8, device=DEV)
        com = torch.zeros(n, dtype=torch.int64, device=DEV)
        bar = torch.zeros(n, dtype=torch.int32, device=DEV)
        rs.set_variant(v)
        rs.accept_step_fused(data, data_len, par, planes, THRESH, com, bar)
        torch.cuda.synchronize()
        res[v] = (par, com, bar, rs.last_kernel())
    rs.set_variant(0)
    assert res[BULK][3] == "rs32_accept_bulk_kernel+tally" and res[0][3] == "rs32_encode_row_kernel+tally"
    for i in range(3):
        assert torch.equal(res[BULK][i], res[0][i])
    idx = torch.arange(0, n, n // 1024, device=DEV)
    want = oracle.rs_encode_uniform(D, P, data[idx].cpu().numpy(), data_len)
    assert (res[BULK][0][:, idx].cpu().numpy() == want).all()
    cw, bw = oracle.tally_planes(planes[:, idx].cpu().numpy().view(np.uint64), THRESH)
    assert (res[BULK][1][idx].cpu().numpy().view(np.uint64) == cw).all()
    assert (res[BULK][2][idx].cpu().numpy().view(np.uint32) == bw).all()


def test_bulk_dispatch(ctx):
    """which kernel each case takes: the bulk kernel only when bit 18 selects it, for the local-plane accept step up to
    256 columns; every other variant keeps its kernel"""
    rs = ReedSolomon(ctx, D, P)

    def kernel(variant, data_len, n=64, flags=SS_RS_OUT_PADDED16, stride=None):
        stride = stride or round_up(data_len, 16)
        data = torch.zeros((n, stride), dtype=torch.uint8, device=DEV)
        L, ds, ps = rs.parity_layout(data_len, n)
        par = torch.zeros(((D + P) * n * ds,), dtype=torch.uint8, device=DEV)
        rs.set_variant(variant)
        check(ctx.lib.ss_rs_encode_uniform_dev(rs.h, data.data_ptr(), stride, data_len, n, par.data_ptr() + D * n * ds,
                                               n * ds, ds, flags))
        torch.cuda.synchronize()
        rs.set_variant(0)
        return rs.last_kernel()

    assert kernel(BULK, 4096) == "rs32_accept_bulk_kernel"
    assert kernel(BULK, 12288) == "rs32_accept_bulk_kernel"
    assert kernel(BULK | (3 << 19) | (1 << 21), 4096) == "rs32_accept_bulk_kernel"            # tuning bits
    assert kernel(BULK, 12289) == "rs32_encode_row_kernel<segmented>"
    assert kernel(0, 4096) == "rs32_encode_row_kernel"
    assert kernel(1, 4096) == kernel(BULK | 1, 4096) == "rs32_encode_uniform_kernel"
    for v in (2, 3, 6, 7, 1 << 4, 1 << 5, 1 << 8, 1 << 10):
        assert kernel(v, 4096) == "rs32_encode_row_kernel", v
    assert kernel(BULK, 4096, flags=SS_RS_OUT_PADDED16 | 2) == "rs32_encode_row_kernel"       # SS_RS_EMIT_DATA
    assert kernel(BULK, 4096, flags=0) == "rs32_encode_uniform_kernel"                        # byte-exact layout
    assert kernel(BULK, 4100, stride=4104) == "rs32_encode_uniform_kernel"                     # stride not 16-aligned
