"""Pins the CPU oracle (oracle/ss_oracle.c) before anything trusts it.

Three groups of checks:
 1. every assertion of the reference's own unit tests for this path, restated on the oracle:
    src/utils/rscoding.rs:685-877 (geometry, null, verify-after-encode, reconstruct, get_data);
 2. the published algorithm of the un-vendored crate `reed-solomon-erasure ^6.0` (Cargo.toml:43):
    field constants, the Backblaze (4,2) matrix, and the crate's / JavaReedSolomon's upstream
    known-answer tests -- RECALLED from the upstream test-suites (galois tests; `test_one_encode`),
    not present in the reference tree, hence "parity unpinned by the reference tree";
 3. the derived KAT of SURVEY.md 8c (TestData("interesting_value"), RS(3,2)).
"""
import itertools

import numpy as np
import pytest


# ---------------------------------------------------------------------------------------------
# 2. crate algorithm
# ---------------------------------------------------------------------------------------------
def test_gf_constants(oracle):
    L = oracle.lib()
    assert [L.ssor_gf_exp_table(i) for i in range(10)] == [1, 2, 4, 8, 16, 32, 64, 128, 29, 58]
    assert [L.ssor_gf_log(i) for i in range(2, 9)] == [1, 25, 2, 50, 26, 198, 3]
    # poly 0x11D: x^8 = x^4+x^3+x^2+1
    assert oracle.gf_mul(0x80, 2) == 0x1D


def test_gf_upstream_kats(oracle):
    """Upstream crate / Backblaze Galois tests (recalled): multiply and exp known answers."""
    assert oracle.gf_mul(3, 4) == 12
    assert oracle.gf_mul(7, 7) == 21
    assert oracle.gf_mul(23, 45) == 41
    assert oracle.gf_exp(2, 2) == 4
    assert oracle.gf_exp(5, 20) == 235
    assert oracle.gf_exp(13, 7) == 43


def test_gf_field_axioms(oracle):
    rng = np.random.default_rng(1)
    for _ in range(2000):
        a, b, c = (int(x) for x in rng.integers(0, 256, 3))
        assert oracle.gf_mul(a, b) == oracle.gf_mul(b, a)
        assert oracle.gf_mul(a, oracle.gf_mul(b, c)) == oracle.gf_mul(oracle.gf_mul(a, b), c)
        assert oracle.gf_mul(a, b ^ c) == oracle.gf_mul(a, b) ^ oracle.gf_mul(a, c)
    for a in range(1, 256):
        assert oracle.gf_mul(a, oracle.lib().ssor_gf_div(1, a)) == 1


def test_matrices(oracle):
    """SURVEY.md 8c table; (4,2) is the well-known Backblaze / klauspost matrix."""
    def rows(d, p):
        return [bytes(r).hex() for r in oracle.rs_matrix(d, p)[d:]]
    assert rows(4, 2) == ["1b1c1214", "1c1b1412"]
    assert rows(3, 2) == ["010101", "0f0806"]
    assert rows(4, 3) == ["1b1c1214", "1c1b1412", "12141b1c"]
    assert rows(5, 4) == ["0707060601", "0908090801", "0f0e0e0f01", "027d95fd16"]
    for d, p in [(1, 1), (2, 1), (3, 2), (6, 4), (9, 6), (12, 8), (17, 3)]:
        m = oracle.rs_matrix(d, p)
        assert (m[:d] == np.eye(d, dtype=np.uint8)).all()          # systematic


def test_upstream_one_encode(oracle):
    """crate `test_one_encode` / JavaReedSolomon `testOneEncode` (5 data + 5 parity), recalled."""
    shards = [np.array(x, dtype=np.uint8) for x in ([0, 1], [4, 5], [2, 3], [6, 7], [8, 9])]
    shards += [np.zeros(2, dtype=np.uint8) for _ in range(5)]
    assert oracle.rs_encode(5, 5, shards) == 0
    assert [s.tolist() for s in shards[5:]] == [[12, 13], [10, 11], [14, 15], [90, 91], [94, 95]]
    rc, ok = oracle.rs_verify(5, 5, shards)
    assert rc == 0 and ok
    shards[8][0] += 1
    rc, ok = oracle.rs_verify(5, 5, shards)
    assert rc == 0 and not ok


def test_new_error_codes(oracle):
    """ReedSolomon::new(d,p): d==0 / p==0 / d+p>256 (SURVEY.md 8c)."""
    assert oracle.rs_new_rc(0, 1) == -3
    assert oracle.rs_new_rc(3, 0) == -5
    assert oracle.rs_new_rc(200, 57) == -2
    assert oracle.rs_new_rc(3, 2) == 0


def test_mds_every_submatrix_invertible(oracle):
    for d, p in [(3, 2), (4, 3), (5, 4)]:
        for keep in itertools.combinations(range(d + p), d):
            present = [1 if i in keep else 0 for i in range(d + p)]
            rc, src, dec = oracle.decode_matrix(d, p, present)
            assert rc == 0 and list(src) == list(keep)


# ---------------------------------------------------------------------------------------------
# 3. derived KAT
# ---------------------------------------------------------------------------------------------
INTERESTING = bytes([17]) + b"interesting_value"      # bincode(TestData("interesting_value")), rscoding.rs:698


def test_interesting_value_kat(oracle):
    sh = oracle.cw_split(INTERESTING, 3)
    assert [bytes(s).hex() for s in sh] == ["11696e746572", "657374696e67", "5f76616c7565"]
    shards = [sh[0].copy(), sh[1].copy(), sh[2].copy(), np.zeros(6, np.uint8), np.zeros(6, np.uint8)]
    assert oracle.rs_encode(3, 2, shards) == 0
    assert bytes(shards[3]).hex() == "2b6c7b717e70"
    assert bytes(shards[4]).hex() == "2ffb9ccc5da8"
    rc, src, dec = oracle.decode_matrix(3, 2, [0, 1, 0, 1, 1])
    assert rc == 0 and list(src) == [1, 3, 4]
    assert [bytes(r).hex() for r in dec] == ["f5699d", "010000", "f4689d"]


# ---------------------------------------------------------------------------------------------
# 1. the reference's own tests, on the oracle
# ---------------------------------------------------------------------------------------------
def _codeword(oracle, data: bytes, d: int, p: int):
    sh = oracle.cw_split(data, d)
    return [sh[i].copy() for i in range(d)] + [None] * p


def test_ref_new_from_data_geometry(oracle):
    """rscoding.rs:697-736"""
    data_len = len(INTERESTING)
    assert data_len == 18
    L = data_len // 3 if data_len % 3 == 0 else data_len // 3 + 1
    assert oracle.cw_shard_len(data_len, 3) == L == 6
    for n in range(0, 200):
        for d in (1, 2, 3, 4, 5, 7):
            assert oracle.cw_shard_len(n, d) == -(-n // d)
    sh = oracle.cw_split(INTERESTING, 3)
    assert sh.shape == (3, 6) and bytes(sh.reshape(-1))[:18] == INTERESTING
    sh = oracle.cw_split(INTERESTING, 4)                       # 18 -> L=5, padded 20
    assert sh.shape == (4, 5) and bytes(sh.reshape(-1)) == INTERESTING + b"\0\0"


def test_ref_compute_verify(oracle):
    """rscoding.rs:788-818 (coder-level part)"""
    cw = _codeword(oracle, INTERESTING, 3, 2)
    cw[3] = np.zeros(6, np.uint8); cw[4] = np.zeros(6, np.uint8)
    assert oracle.rs_encode(3, 2, cw) == 0
    rc, ok = oracle.rs_verify(3, 2, cw)
    assert rc == 0 and ok


def test_ref_reconstruction(oracle):
    """rscoding.rs:820-862"""
    full = _codeword(oracle, INTERESTING, 3, 2)
    # parity missing -> reconstruct_all regenerates them
    cw = [s if s is None else s.copy() for s in full]
    assert oracle.rs_reconstruct(3, 2, cw, False) == 0 and all(s is not None for s in cw)
    golden = [s.copy() for s in cw]
    # erase {1,3}
    cw[1] = None; cw[3] = None
    assert oracle.rs_reconstruct(3, 2, cw, False) == 0
    assert all((a == b).all() for a, b in zip(cw, golden))
    # erase {0,2}, data only
    cw[0] = None; cw[2] = None
    assert oracle.rs_reconstruct(3, 2, cw, True) == 0
    assert all((a == b).all() for a, b in zip(cw[:3], golden[:3]))
    # 3 of 5 missing -> error, never partial
    cw[0] = None; cw[1] = None; cw[4] = None
    assert oracle.rs_reconstruct(3, 2, cw, False) == -10
    assert oracle.rs_reconstruct(3, 2, cw, True) == -10
    assert cw[0] is None and cw[1] is None and cw[4] is None


def test_ref_get_data_roundtrip(oracle):
    """rscoding.rs:864-876"""
    cw = _codeword(oracle, INTERESTING, 3, 2)
    cw[3] = np.zeros(6, np.uint8); cw[4] = np.zeros(6, np.uint8)
    oracle.rs_encode(3, 2, cw)
    cw[0] = None
    assert oracle.rs_reconstruct(3, 2, cw, True) == 0
    assert bytes(np.concatenate(cw[:3]))[:18] == INTERESTING


@pytest.mark.parametrize("d,p", [(3, 2), (4, 3), (5, 4), (2, 1), (6, 4)])
def test_roundtrip_all_erasure_patterns(oracle, d, p):
    rng = np.random.default_rng(d * 100 + p)
    data = rng.integers(0, 256, 97, dtype=np.uint8).tobytes()
    base = _codeword(oracle, data, d, p)
    L = len(base[0])
    for j in range(p):
        base[d + j] = np.zeros(L, np.uint8)
    assert oracle.rs_encode(d, p, base) == 0
    for nmiss in range(1, p + 1):
        for miss in itertools.combinations(range(d + p), nmiss):
            cw = [None if i in miss else base[i].copy() for i in range(d + p)]
            assert oracle.rs_reconstruct(d, p, cw, False) == 0
            assert all((a == b).all() for a, b in zip(cw, base))


def test_batch_matches_single_and_simd(oracle):
    rng = np.random.default_rng(7)
    for d, p, dl in [(3, 2, 4096), (3, 2, 1), (3, 2, 17), (4, 3, 1000), (5, 4, 333)]:
        n = 9
        stride = (dl + 15) // 16 * 16 + 16
        data = rng.integers(0, 256, (n, stride), dtype=np.uint8)
        par0 = oracle.rs_encode_uniform(d, p, data, dl, mode=0, threads=1)
        par1 = oracle.rs_encode_uniform(d, p, data, dl, mode=1, threads=2)
        assert (par0 == par1).all()
        L = oracle.cw_shard_len(dl, d)
        for g in range(n):
            cw = _codeword(oracle, data[g, :dl].tobytes(), d, p)
            for j in range(p):
                cw[d + j] = np.zeros(L, np.uint8)
            oracle.rs_encode(d, p, cw)
            for j in range(p):
                assert (par0[j, g, :L] == cw[d + j]).all()
                assert (par0[j, g, L:] == 0).all()


def test_oracle_reproduces_committed_golden_fixtures(oracle):
    """tests/golden/*.npz were generated by tests/golden/make_golden.py from this oracle; any drift of the oracle
    (or of the seeded workload generators) shows up here on the CPU, before a GPU is involved."""
    from pathlib import Path
    z = np.load(Path(__file__).parent / "golden" / "rs_golden.npz")
    keys = [k[5:] for k in z.files if k.startswith("data_")]
    assert len(keys) >= 6
    for key in keys:
        d, p, data_len = (int(x) for x in key.split("_"))
        assert (oracle.rs_encode_uniform(d, p, z["data_" + key], data_len) == z["parity_" + key]).all(), key
    t = np.load(Path(__file__).parent / "golden" / "tally_golden.npz")
    c, bar = oracle.tally_planes(t["planes"], int(t["threshold"]))
    assert (c == t["committed"]).all() and (bar == t["commit_bar"]).all()
    nc = oracle.raft_scan_batch(t["raft_match"], t["raft_last_commit"], t["raft_log_end"], t["raft_curr_term"],
                                t["raft_terms"], int(t["raft_threshold"]))
    assert (nc == t["raft_new_commit"]).all()


def test_cargo_vectors_file_is_what_the_oracle_produces(oracle):
    """tests/golden/rs_vectors.json is the input of tests/golden/verify_with_cargo.rs (the pin a maintainer with Rust can
    run).  Guard it against drift: every vector must be what the oracle produces today, the hand-written bincode of the
    real request batch must decode back to its fields, and its frames must parse to the same codeword."""
    import json
    from pathlib import Path
    vec = json.loads((Path(__file__).parent / "golden" / "rs_vectors.json").read_text())
    for case in vec["rs"]:
        d, p, dl = case["d"], case["p"], case["data_len"]
        payload = bytes.fromhex(case["payload"])
        assert len(payload) == dl
        L = oracle.cw_shard_len(dl, d)
        row = np.zeros((1, (dl + 15) // 16 * 16), dtype=np.uint8)
        row[0, :dl] = np.frombuffer(payload, dtype=np.uint8)
        par = oracle.rs_encode_uniform(d, p, row, dl)
        assert [bytes(s).hex() for s in oracle.cw_split(payload, d)] == case["data_shards"]
        assert [par[j, 0, :L].tobytes().hex() for j in range(p)] == case["parity_shards"]
    for case in vec["bitmap"]:
        bits = sum(1 << i for i in case["ones"])
        assert oracle.bitmap_encode(case["size"], bits).hex() == case["bincode"]
    g = vec["reqbatch_put"]
    b = bytes.fromhex(g["bincode"])
    # bincode 2 standard(): Vec len, ClientId, variant Req, id, variant Put, key, value -- all below 251, one byte each
    assert b[:5] == bytes([1, 7, 0, 1, 1]) and b[5] == 2 and b[6:8] == b"k1" and b[8] == 22 and b[9:] == b"value-0123456789abcdef"
    assert g["data_len"] == len(b) == 31 and g["shard_len"] == 11
    shards = [bytes.fromhex(s) for s in g["shards"]]
    assert b"".join(shards[:3]) == b + bytes(2)                       # contiguous split, zero-padded tail
    full = [np.frombuffer(s, dtype=np.uint8).copy() for s in shards]
    assert oracle.rs_verify(3, 2, full) == (0, True)
    for key, kind in (("accept_frame_shard1_slot300_ballot70000", 0), ("wal_accept_data_shard1_slot300_ballot70000", 1)):
        dec = oracle.decode_accept(bytes.fromhex(g[key]), kind)
        assert dec is not None and (dec["slot"], dec["ballot"], dec["d"], dec["p"], dec["data_len"], dec["shard_len"]) == (300, 70000, 3, 2, 31, 11)
        assert [s is not None for s in dec["shards"]] == [False, True, False, False, False] and dec["shards"][1] == shards[1]
    dec = oracle.decode_accept(bytes.fromhex(g["crossword_accept_frame_shards12_slot300_ballot70000_assignment_spr2"]), 0, with_assignment=True)
    assert dec["shards"][1] == shards[1] and dec["shards"][2] == shards[2] and dec["assignment"] == [3, 6, 12, 24, 17] and dec["assign_size"] == 5
