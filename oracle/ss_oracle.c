/*
 * ss_oracle.c -- CPU ORACLE (test infrastructure; see ss_oracle.h for scope and pinning status).
 *
 * Restates, in plain C, the algorithms on the reference's quorum-tally + Reed-Solomon path.
 * Every function cites the reference file:line (relative to the reference tree's root) it follows.
 * Build: `make -C oracle` (gcc -O3 -fopenmp; SIMD paths use per-function target attributes and
 * a runtime CPU check, so the .so stays runnable on a host without AVX2).
 */
#include "ss_oracle.h"

#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif
#if defined(__x86_64__)
#include <immintrin.h>
#endif

/* ------------------------------------------------------------------------------------------
 * GF(2^8): crate reed-solomon-erasure galois_8 (used at src/utils/rscoding.rs:9).
 * Generating polynomial 0x11D (x^8+x^4+x^3+x^2+1), generator element 2.
 * ------------------------------------------------------------------------------------------ */
static uint8_t GF_EXP[512];
static uint8_t GF_LOG[256];
static uint8_t GF_MUL[256][256];
static uint8_t GF_MUL_LO[256][16]; /* c * n         (low nibble products)  */
static uint8_t GF_MUL_HI[256][16]; /* c * (n << 4)  (high nibble products) */
static int gf_ready = 0;

static void gf_init(void) {
    if (gf_ready) return;
    unsigned x = 1;
    for (unsigned i = 0; i < 255; i++) {
        GF_EXP[i] = (uint8_t)x;
        GF_LOG[x] = (uint8_t)i;
        x <<= 1;
        if (x & 0x100) x ^= 0x11D;
    }
    for (unsigned i = 255; i < 512; i++) GF_EXP[i] = GF_EXP[i - 255];
    GF_LOG[0] = 0; /* undefined; never read for a == 0 */
    for (unsigned a = 0; a < 256; a++)
        for (unsigned b = 0; b < 256; b++)
            GF_MUL[a][b] = (a == 0 || b == 0) ? 0 : GF_EXP[GF_LOG[a] + GF_LOG[b]];
    for (unsigned c = 0; c < 256; c++)
        for (unsigned n = 0; n < 16; n++) {
            GF_MUL_LO[c][n] = GF_MUL[c][n];
            GF_MUL_HI[c][n] = GF_MUL[c][n << 4];
        }
    gf_ready = 1;
}

__attribute__((constructor)) static void ssor_ctor(void) { gf_init(); }

uint8_t ssor_gf_mul(uint8_t a, uint8_t b) { gf_init(); return GF_MUL[a][b]; }
uint8_t ssor_gf_log(uint8_t a) { gf_init(); return GF_LOG[a]; }
uint8_t ssor_gf_exp_table(unsigned i) { gf_init(); return GF_EXP[i % 510]; }

uint8_t ssor_gf_div(uint8_t a, uint8_t b) {
    gf_init();
    if (a == 0) return 0;
    int l = (int)GF_LOG[a] - (int)GF_LOG[b];
    if (l < 0) l += 255;
    return GF_EXP[l];
}

/* crate galois_8::exp(a, n): n == 0 -> 1; a == 0 -> 0; else EXP[(LOG[a]*n) mod 255] */
uint8_t ssor_gf_exp(uint8_t a, unsigned n) {
    gf_init();
    if (n == 0) return 1;
    if (a == 0) return 0;
    unsigned l = ((unsigned)GF_LOG[a] * n) % 255u;
    return GF_EXP[l];
}

/* ------------------------------------------------------------------------------------------
 * Matrix construction (crate ReedSolomon::build_matrix, a port of Backblaze JavaReedSolomon):
 *   V = vandermonde(d+p, d), V[r][c] = exp(r, c);  M = V * inverse(V[0..d]).
 * Constructors in the reference: rspaxos/mod.rs:606, crossword/mod.rs:827, craft/mod.rs:534.
 * ------------------------------------------------------------------------------------------ */
int ssor_gf_matrix_invert(int n, const uint8_t *in, uint8_t *out) {
    gf_init();
    if (n <= 0 || n > 256) return SSOR_ERR_INVALID_ARG;
    int w = 2 * n;
    uint8_t *a = (uint8_t *)calloc((size_t)n * w, 1);
    if (!a) return SSOR_ERR_INVALID_ARG;
    for (int r = 0; r < n; r++) {
        memcpy(a + (size_t)r * w, in + (size_t)r * n, n);
        a[(size_t)r * w + n + r] = 1;
    }
    /* Gaussian elimination: pivot search downward, scale, clear below; then clear above */
    for (int r = 0; r < n; r++) {
        if (a[(size_t)r * w + r] == 0) {
            int rb = r + 1;
            while (rb < n && a[(size_t)rb * w + r] == 0) rb++;
            if (rb == n) { free(a); return SSOR_ERR_SINGULAR; }
            for (int c = 0; c < w; c++) {
                uint8_t t = a[(size_t)r * w + c];
                a[(size_t)r * w + c] = a[(size_t)rb * w + c];
                a[(size_t)rb * w + c] = t;
            }
        }
        uint8_t piv = a[(size_t)r * w + r];
        if (piv != 1) {
            uint8_t s = ssor_gf_div(1, piv);
            for (int c = 0; c < w; c++) a[(size_t)r * w + c] = GF_MUL[a[(size_t)r * w + c]][s];
        }
        for (int rb = r + 1; rb < n; rb++) {
            uint8_t s = a[(size_t)rb * w + r];
            if (s != 0)
                for (int c = 0; c < w; c++)
                    a[(size_t)rb * w + c] ^= GF_MUL[s][a[(size_t)r * w + c]];
        }
    }
    for (int dcol = 0; dcol < n; dcol++)
        for (int ra = 0; ra < dcol; ra++) {
            uint8_t s = a[(size_t)ra * w + dcol];
            if (s != 0)
                for (int c = 0; c < w; c++)
                    a[(size_t)ra * w + c] ^= GF_MUL[s][a[(size_t)dcol * w + c]];
        }
    for (int r = 0; r < n; r++) memcpy(out + (size_t)r * n, a + (size_t)r * w + n, n);
    free(a);
    return SSOR_OK;
}

static int rs_check_dp(int d, int p) {
    /* crate ReedSolomon::new: d == 0 -> TooFewDataShards; p == 0 -> TooFewParityShards;
     * d + p > 256 -> TooManyShards.  (Summerset special-cases p == 0 before touching the
     * coder: rscoding.rs:454-456,498-507.) */
    if (d <= 0) return SSOR_ERR_TOO_FEW_DATA_SHARDS;
    if (p <= 0) return SSOR_ERR_TOO_FEW_PARITY_SHARDS;
    if (d + p > 256) return SSOR_ERR_TOO_MANY_SHARDS;
    return SSOR_OK;
}

int ssor_rs_build_matrix(int d, int p, uint8_t *out) {
    int rc = rs_check_dp(d, p);
    if (rc) return rc;
    int t = d + p;
    uint8_t *v = (uint8_t *)malloc((size_t)t * d);
    uint8_t *top = (uint8_t *)malloc((size_t)d * d);
    uint8_t *inv = (uint8_t *)malloc((size_t)d * d);
    for (int r = 0; r < t; r++)
        for (int c = 0; c < d; c++) v[(size_t)r * d + c] = ssor_gf_exp((uint8_t)r, (unsigned)c);
    memcpy(top, v, (size_t)d * d);
    rc = ssor_gf_matrix_invert(d, top, inv);
    if (rc == SSOR_OK)
        for (int r = 0; r < t; r++)
            for (int c = 0; c < d; c++) {
                uint8_t acc = 0;
                for (int k = 0; k < d; k++) acc ^= GF_MUL[v[(size_t)r * d + k]][inv[(size_t)k * d + c]];
                out[(size_t)r * d + c] = acc;
            }
    free(v); free(top); free(inv);
    return rc;
}

int ssor_rs_decode_matrix(int d, int p, const uint8_t *present, int *src_idx, uint8_t *dec) {
    int rc = rs_check_dp(d, p);
    if (rc) return rc;
    int t = d + p, k = 0;
    for (int i = 0; i < t && k < d; i++)
        if (present[i]) src_idx[k++] = i;
    if (k < d) return SSOR_ERR_TOO_FEW_SHARDS_PRESENT;
    uint8_t *m = (uint8_t *)malloc((size_t)t * d);
    uint8_t *sub = (uint8_t *)malloc((size_t)d * d);
    ssor_rs_build_matrix(d, p, m);
    for (int r = 0; r < d; r++) memcpy(sub + (size_t)r * d, m + (size_t)src_idx[r] * d, d);
    rc = ssor_gf_matrix_invert(d, sub, dec);
    free(m); free(sub);
    return rc;
}

/* ------------------------------------------------------------------------------------------
 * Byte loops.  Scalar: out[k] (^)= MUL_TABLE[c][in[k]] (crate mul_slice / mul_slice_xor).
 * AVX2: 16-entry low/high nibble tables + vpshufb (what the crate's `simd-accel` C code does;
 * enabled by Summerset's `rse-simd` feature, Cargo.toml:57-58, scripts/utils/file.py:33).
 * ------------------------------------------------------------------------------------------ */
static void mul_slice_scalar(uint8_t c, const uint8_t *in, uint8_t *out, size_t n, int xor_into) {
    const uint8_t *row = GF_MUL[c];
    if (xor_into) for (size_t k = 0; k < n; k++) out[k] ^= row[in[k]];
    else          for (size_t k = 0; k < n; k++) out[k] = row[in[k]];
}

#if defined(__x86_64__)
__attribute__((target("avx2")))
static void mul_slice_avx2(uint8_t c, const uint8_t *in, uint8_t *out, size_t n, int xor_into) {
    const __m256i lo = _mm256_broadcastsi128_si256(_mm_loadu_si128((const __m128i *)GF_MUL_LO[c]));
    const __m256i hi = _mm256_broadcastsi128_si256(_mm_loadu_si128((const __m128i *)GF_MUL_HI[c]));
    const __m256i m4 = _mm256_set1_epi8(0x0f);
    size_t k = 0;
    for (; k + 32 <= n; k += 32) {
        __m256i x = _mm256_loadu_si256((const __m256i *)(in + k));
        __m256i l = _mm256_shuffle_epi8(lo, _mm256_and_si256(x, m4));
        __m256i h = _mm256_shuffle_epi8(hi, _mm256_and_si256(_mm256_srli_epi64(x, 4), m4));
        __m256i r = _mm256_xor_si256(l, h);
        if (xor_into) r = _mm256_xor_si256(r, _mm256_loadu_si256((const __m256i *)(out + k)));
        _mm256_storeu_si256((__m256i *)(out + k), r);
    }
    if (k < n) mul_slice_scalar(c, in + k, out + k, n - k, xor_into);
}
#endif

int ssor_have_avx2(void) {
#if defined(__x86_64__)
    return __builtin_cpu_supports("avx2") ? 1 : 0;
#else
    return 0;
#endif
}

int ssor_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

static void mul_slice(uint8_t c, const uint8_t *in, uint8_t *out, size_t n, int xor_into, int mode) {
#if defined(__x86_64__)
    if (mode == 1) { mul_slice_avx2(c, in, out, n, xor_into); return; }
#endif
    (void)mode;
    mul_slice_scalar(c, in, out, n, xor_into);
}

/* out_j = sum_i rows[j][i] * in_i  (crate code_some_slices: first input assigns, rest XOR) */
static void code_some(const uint8_t *rows, int n_in, const uint8_t *const *in, int n_out,
                      uint8_t *const *out, size_t len, int mode) {
    for (int j = 0; j < n_out; j++)
        for (int i = 0; i < n_in; i++)
            mul_slice(rows[(size_t)j * n_in + i], in[i], out[j], len, i != 0, mode);
}

static int resolve_mode(int mode) { return (mode == 1 && ssor_have_avx2()) ? 1 : 0; }

/* crate ReedSolomon::encode, called from RSCodeword::compute_parity (rscoding.rs:484) */
int ssor_rs_encode(int d, int p, uint8_t *const *shards, size_t shard_len) {
    int rc = rs_check_dp(d, p);
    if (rc) return rc;
    if (shard_len == 0) return SSOR_ERR_EMPTY_SHARD;
    uint8_t *m = (uint8_t *)malloc((size_t)(d + p) * d);
    ssor_rs_build_matrix(d, p, m);
    code_some(m + (size_t)d * d, d, (const uint8_t *const *)shards, p, shards + d, shard_len, 0);
    free(m);
    return SSOR_OK;
}

/* crate ReedSolomon::reconstruct / reconstruct_data, called from rscoding.rs:515,517.
 * Picks the first d present shards by index, inverts that sub-matrix, regenerates missing data
 * shards; unless data_only, then re-encodes missing parity from the (now complete) data. */
static int reconstruct_mode(int d, int p, uint8_t *const *shards, uint8_t *present,
                            size_t shard_len, int data_only, int mode) {
    int rc = rs_check_dp(d, p);
    if (rc) return rc;
    int t = d + p, np = 0;
    for (int i = 0; i < t; i++) np += present[i] ? 1 : 0;
    if (np == t) return SSOR_OK;            /* nothing to do */
    if (np < d) return SSOR_ERR_TOO_FEW_SHARDS_PRESENT;
    if (shard_len == 0) return SSOR_ERR_EMPTY_SHARD;

    int src_idx[256];
    uint8_t *dec = (uint8_t *)malloc((size_t)d * d);
    rc = ssor_rs_decode_matrix(d, p, present, src_idx, dec);
    if (rc) { free(dec); return rc; }
    const uint8_t *src[256];
    for (int k = 0; k < d; k++) src[k] = shards[src_idx[k]];
    for (int i = 0; i < d; i++)
        if (!present[i]) {
            uint8_t *o = shards[i];
            code_some(dec + (size_t)i * d, d, src, 1, &o, shard_len, mode);
        }
    free(dec);
    if (!data_only) {
        uint8_t *m = (uint8_t *)malloc((size_t)t * d);
        ssor_rs_build_matrix(d, p, m);
        for (int j = d; j < t; j++)
            if (!present[j]) {
                uint8_t *o = shards[j];
                code_some(m + (size_t)j * d, d, (const uint8_t *const *)shards, 1, &o, shard_len, mode);
            }
        free(m);
    }
    for (int i = 0; i < (data_only ? d : t); i++) present[i] = 1;
    return SSOR_OK;
}

int ssor_rs_reconstruct(int d, int p, uint8_t *const *shards, uint8_t *present,
                        size_t shard_len, int data_only) {
    return reconstruct_mode(d, p, shards, present, shard_len, data_only, 0);
}

/* crate ReedSolomon::verify, called from RSCodeword::verify_parity (rscoding.rs:575) */
int ssor_rs_verify(int d, int p, const uint8_t *const *shards, size_t shard_len, int *ok) {
    int rc = rs_check_dp(d, p);
    if (rc) return rc;
    if (shard_len == 0) return SSOR_ERR_EMPTY_SHARD;
    uint8_t *m = (uint8_t *)malloc((size_t)(d + p) * d);
    uint8_t *buf = (uint8_t *)malloc(shard_len);
    ssor_rs_build_matrix(d, p, m);
    *ok = 1;
    for (int j = 0; j < p && *ok; j++) {
        uint8_t *o = buf;
        code_some(m + (size_t)(d + j) * d, d, shards, 1, &o, shard_len, 0);
        if (memcmp(buf, shards[d + j], shard_len) != 0) *ok = 0;
    }
    free(m); free(buf);
    return SSOR_OK;
}

/* ------------------------------------------------------------------------------------------
 * RSCodeword geometry: rscoding.rs:165-220 (internal_new).
 * ------------------------------------------------------------------------------------------ */
size_t ssor_cw_shard_len(size_t data_len, int d) {
    /* rscoding.rs:177-181 */
    return (data_len % (size_t)d == 0) ? data_len / (size_t)d : data_len / (size_t)d + 1;
}

void ssor_cw_split(const uint8_t *data, size_t data_len, int d, uint8_t *out) {
    /* rscoding.rs:188-199: resize(padded_len, 0) then contiguous split_to(shard_len) */
    size_t L = ssor_cw_shard_len(data_len, d);
    memcpy(out, data, data_len);
    memset(out + data_len, 0, L * (size_t)d - data_len);
}

/* ------------------------------------------------------------------------------------------
 * Batched CPU path: from_data's pad/split + compute_parity per codeword
 * (rspaxos/request.rs:72-77, crossword/request.rs:82-87), OpenMP over codewords.
 * ------------------------------------------------------------------------------------------ */
int ssor_rs_encode_batch(int d, int p, const uint8_t *data, const uint64_t *data_off,
                         const uint32_t *data_len, uint64_t n, uint8_t *parity,
                         uint64_t plane_stride, const uint64_t *par_off, int mode, int threads) {
    int rc = rs_check_dp(d, p);
    if (rc) return rc;
    const int sched_static = mode & SSOR_MODE_STATIC;     /* contiguous block of codewords per thread (NUMA first-touch) */
    mode = resolve_mode(mode & 0xff);
    uint8_t *m = (uint8_t *)malloc((size_t)(d + p) * d);
    ssor_rs_build_matrix(d, p, m);
    const uint8_t *prow = m + (size_t)d * d;
#ifdef _OPENMP
    if (threads <= 0) threads = omp_get_max_threads();
    if (sched_static) omp_set_schedule(omp_sched_static, 0); else omp_set_schedule(omp_sched_dynamic, 256);
#pragma omp parallel num_threads(threads)
#endif
    {
        uint8_t *tail = NULL; size_t tail_cap = 0;
#ifdef _OPENMP
#pragma omp for schedule(runtime)
#endif
        for (uint64_t g = 0; g < n; g++) {
            size_t len = data_len[g];
            if (len == 0) continue;                       /* null codeword: nothing to encode */
            size_t L = ssor_cw_shard_len(len, d);
            const uint8_t *base = data + data_off[g];
            const uint8_t *in[256];
            uint8_t *out[256];
            /* data shard i = bytes [i*L, (i+1)*L); only the last one can need zero padding */
            for (int i = 0; i < d; i++) in[i] = base + (size_t)i * L;
            size_t padded = L * (size_t)d;
            if (padded != len) {
                /* shards whose range crosses data_len get a zero-padded private copy */
                if (tail_cap < padded) { free(tail); tail = (uint8_t *)malloc(padded); tail_cap = padded; }
                int first = (int)(len / L);
                size_t start = (size_t)first * L;
                memcpy(tail + start, base + start, len - start);
                memset(tail + len, 0, padded - len);
                for (int i = first; i < d; i++) in[i] = tail + (size_t)i * L;
            }
            for (int j = 0; j < p; j++) out[j] = parity + (size_t)j * plane_stride + par_off[g];
            code_some(prow, d, in, p, out, L, mode);
        }
        free(tail);
    }
    free(m);
    return SSOR_OK;
}

/* Fills n_items items of item_bytes bytes (item g at buf + g*item_stride) with a seeded byte stream, in the SAME
 * static thread partition SSOR_MODE_STATIC uses for the encode loop, so that on a NUMA host every page is first
 * touched -- hence placed -- on the node of the thread that will later read or write it.  Benchmark plumbing. */
void ssor_first_touch_fill(uint8_t *buf, uint64_t n_items, uint64_t item_bytes, uint64_t item_stride,
                           uint64_t seed, int zero, int threads) {
#ifdef _OPENMP
    if (threads <= 0) threads = omp_get_max_threads();
#pragma omp parallel for schedule(static) num_threads(threads)
#endif
    for (uint64_t g = 0; g < n_items; g++) {
        uint8_t *q = buf + g * item_stride;
        if (zero) { memset(q, 0, item_bytes); continue; }
        uint64_t x = seed ^ (g * 0x9E3779B97F4A7C15ull + 0xD1B54A32D192ED03ull);
        uint64_t i = 0;
        for (; i + 8 <= item_bytes; i += 8) {
            x ^= x << 13; x ^= x >> 7; x ^= x << 17;       /* xorshift64 */
            memcpy(q + i, &x, 8);
        }
        for (; i < item_bytes; i++) { x ^= x << 13; x ^= x >> 7; x ^= x << 17; q[i] = (uint8_t)x; }
    }
}

int ssor_rs_reconstruct_batch(int d, int p, uint8_t *shards, uint64_t plane_stride,
                              const uint64_t *off, const uint32_t *data_len,
                              const uint32_t *present, uint64_t n, int data_only,
                              int32_t *status, int mode, int threads) {
    int rc = rs_check_dp(d, p);
    if (rc) return rc;
    if (d + p > 32) return SSOR_ERR_INVALID_ARG;
    mode = resolve_mode(mode);
    int t = d + p;
#ifdef _OPENMP
    if (threads <= 0) threads = omp_get_max_threads();
#pragma omp parallel for schedule(dynamic, 256) num_threads(threads)
#endif
    for (uint64_t g = 0; g < n; g++) {
        size_t L = ssor_cw_shard_len(data_len[g], d);
        uint8_t *sp[32];
        uint8_t pres[32];
        for (int j = 0; j < t; j++) {
            sp[j] = shards + (size_t)j * plane_stride + off[g];
            pres[j] = (present[g] >> j) & 1u;
        }
        if (data_len[g] == 0) { status[g] = SSOR_ERR_INVALID_ARG; continue; } /* null codeword */
        status[g] = reconstruct_mode(d, p, sp, pres, L, data_only, mode);
    }
    return SSOR_OK;
}

/* ------------------------------------------------------------------------------------------
 * Quorum tallies.
 * ------------------------------------------------------------------------------------------ */
static inline unsigned popc32(uint32_t x) { return (unsigned)__builtin_popcount(x); }

/* multipaxos/messages.rs:370-443 (rspaxos/messages.rs:395-465 identical up to threshold).
 * The leader's own ack enters through the same function (multipaxos/durability.rs:99-103):
 * callers put the leader's id in the record stream like any other peer.
 * `slot < start_slot` (messages.rs:377) cannot occur in a fixed S-slot window (start_slot = 0);
 * `is_leader` is true for every group by construction (leader-side state only). */
void ssor_tally_stream(const uint32_t *rec_g, const uint8_t *rec_s, const uint8_t *rec_p,
                       const uint64_t *rec_b, uint64_t n_rec, uint32_t S, uint32_t population,
                       uint32_t threshold, const uint64_t *bal_prepared, const uint64_t *inst_bal,
                       uint8_t *status, uint16_t *acks) {
    for (uint64_t i = 0; i < n_rec; i++) {
        uint32_t g = rec_g[i];
        uint32_t s = rec_s[i], peer = rec_p[i];
        uint64_t ballot = rec_b[i];
        if (ballot != bal_prepared[g]) continue;                    /* :388 */
        uint64_t k = (uint64_t)g * S + s;
        if (status[k] != SSOR_ST_ACCEPTING || ballot < inst_bal[k]) continue; /* :394-399 */
        if (peer >= population) continue;                           /* Bitmap::get Err, bitmap.rs:89-97 */
        if (acks[k] & (1u << peer)) continue;                       /* :404-406 duplicate */
        acks[k] |= (uint16_t)(1u << peer);                          /* :409 */
        if (popc32(acks[k]) >= threshold) status[k] = SSOR_ST_COMMITTED; /* :412-413 */
    }
}

/* crossword/messages.rs:481-574: the same handler with the Crossword commit condition.  The ack set is
 * HashMap<peer, assignment[peer]>: a peer bitmask plus the instance's assignment (policies[policy_idx[k]]). */
void ssor_tally_stream_crossword(const uint32_t *rec_g, const uint8_t *rec_s, const uint8_t *rec_p,
                                 const uint64_t *rec_b, uint64_t n_rec, uint32_t S, uint32_t population,
                                 uint32_t T, uint32_t d, uint32_t majority, uint32_t f, int balanced,
                                 const uint32_t *policies, uint32_t n_policies, const uint8_t *policy_idx,
                                 const uint64_t *bal_prepared, const uint64_t *inst_bal, uint8_t *status,
                                 uint16_t *acks) {
    for (uint64_t i = 0; i < n_rec; i++) {
        uint32_t g = rec_g[i];
        uint32_t s = rec_s[i], peer = rec_p[i];
        uint64_t ballot = rec_b[i];
        if (ballot != bal_prepared[g]) continue;                    /* :500 */
        uint64_t k = (uint64_t)g * S + s;
        if (status[k] != SSOR_ST_ACCEPTING || ballot < inst_bal[k]) continue; /* :513-519 */
        if (peer >= population) continue;                           /* assignment[peer] would be out of range */
        if (acks[k] & (1u << peer)) continue;                       /* :524-526 contains_key */
        acks[k] |= (uint16_t)(1u << peer);                          /* :529-531 */
        if (policy_idx[k] >= n_policies) continue;
        if (ssor_cw_committed(T, population, d, majority, f, acks[k],
                              policies + (size_t)policy_idx[k] * population, balanced))
            status[k] = SSOR_ST_COMMITTED;                          /* :535-544 */
    }
}

uint32_t ssor_commit_bar(uint64_t w) {
    /* multipaxos/durability.rs:161-170: advance while status >= Committed */
    uint32_t bar = 0;
    while (bar < 64 && ((w >> bar) & 1ull)) bar++;
    return bar;
}

void ssor_tally_planes(const uint64_t *planes, uint32_t R, uint64_t G, uint32_t threshold,
                       uint64_t *committed, uint32_t *commit_bar, int threads) {
#ifdef _OPENMP
    if (threads <= 0) threads = omp_get_max_threads();
#pragma omp parallel for schedule(static) num_threads(threads)
#endif
    for (uint64_t g = 0; g < G; g++) {
        uint64_t w = 0;
        for (unsigned s = 0; s < 64; s++) {
            unsigned cnt = 0;                       /* Bitmap::count(), bitmap.rs:111-113 */
            for (uint32_t r = 0; r < R; r++) cnt += (unsigned)((planes[(uint64_t)r * G + g] >> s) & 1ull);
            if (cnt >= threshold) w |= (1ull << s);
        }
        committed[g] = w;
        if (commit_bar) commit_bar[g] = ssor_commit_bar(w);
    }
}

void ssor_tally_masks(const uint16_t *masks, uint64_t n, uint32_t threshold, uint8_t *commit) {
    for (uint64_t i = 0; i < n; i++) commit[i] = popc32(masks[i]) >= threshold ? 1 : 0;
}

/* ------------------------------------------------------------------------------------------
 * Crossword.
 * ------------------------------------------------------------------------------------------ */
void ssor_cw_brr_assignment(uint32_t n, uint32_t T, uint32_t spr, uint32_t *out) {
    /* crossword/mod.rs:866-888: ((r*dj)..(r*dj+spr)).map(|i| i % T) */
    uint32_t dj = T / n;
    for (uint32_t r = 0; r < n; r++) {
        uint32_t m = 0;
        for (uint32_t i = r * dj; i < r * dj + spr; i++) m |= 1u << (i % T);
        out[r] = m;
    }
}

uint32_t ssor_cw_min_spr(uint32_t d, uint32_t majority, uint32_t f, uint32_t alive) {
    /* crossword/adaptive.rs:98-106 */
    return (majority + f + 1 - alive) * (d / majority);
}

uint32_t ssor_cw_coverage(uint32_t T, uint32_t n, uint32_t ack_mask, const uint32_t *assignment,
                          uint32_t f, int balanced) {
    /* crossword/messages.rs:15-62 */
    uint32_t servers[32], ns = 0;
    for (uint32_t r = 0; r < n; r++)
        if (ack_mask & (1u << r)) servers[ns++] = r;
    if (ns <= f) return 0;                                      /* :22-24 */
    if (balanced) {                                             /* :28-33 */
        uint32_t spr = popc32(assignment[servers[0]]);
        uint32_t dj = T / n;
        return (ns - f - 1) * dj + spr;
    }
    uint32_t cnt = ns - f, min_cov = T;                         /* :35-61 */
    for (uint32_t sub = 0; sub < (1u << ns); sub++) {
        if (popc32(sub) != cnt) continue;
        uint32_t cov = 0;
        for (uint32_t i = 0; i < ns; i++)
            if ((sub >> i) & 1u) cov |= assignment[servers[i]];
        uint32_t c = popc32(cov);
        if (c < min_cov) min_cov = c;
    }
    return min_cov;
}

int ssor_cw_committed(uint32_t T, uint32_t n, uint32_t d, uint32_t majority, uint32_t f,
                      uint32_t ack_mask, const uint32_t *assignment, int balanced) {
    /* crossword/messages.rs:535-542 */
    uint32_t na = popc32(ack_mask & ((n >= 32) ? 0xffffffffu : ((1u << n) - 1u)));
    return na >= majority && ssor_cw_coverage(T, n, ack_mask, assignment, f, balanced) >= d;
}

/* ------------------------------------------------------------------------------------------
 * Raft commit scan: raft/messages.rs:256-275 (CRaft: craft/messages.rs:288-314 passes another
 * threshold).  match_slot excludes self (raft/mod.rs:560-562); "1 +" is the leader (:266).
 * ------------------------------------------------------------------------------------------ */
uint32_t ssor_raft_scan(const uint32_t *match, uint32_t npeers, uint32_t last_commit,
                        uint32_t log_end, uint32_t curr_term, const uint32_t *terms,
                        uint32_t threshold) {
    uint32_t new_commit = last_commit;
    for (uint32_t slot = last_commit + 1; slot < log_end; slot++) {
        if (terms[slot - (last_commit + 1)] != curr_term) continue;   /* :261-263 */
        uint32_t cnt = 1;
        for (uint32_t q = 0; q < npeers; q++) cnt += match[q] >= slot ? 1u : 0u; /* :266-270 */
        if (cnt >= threshold) new_commit = slot;                       /* :271-274, no break */
    }
    return new_commit;
}

uint32_t ssor_raft_snap_scan(const uint32_t *match, uint32_t npeers, uint32_t last_snap,
                             uint32_t end_slot) {
    /* raft/messages.rs:298-309 */
    uint32_t snap = last_snap;
    for (uint32_t slot = last_snap + 1; slot <= end_slot; slot++) {
        uint32_t cnt = 1;
        for (uint32_t q = 0; q < npeers; q++) cnt += match[q] >= slot ? 1u : 0u;
        if (cnt == npeers + 1) snap = slot;
    }
    return snap;
}

void ssor_raft_scan_batch(const uint32_t *match, uint32_t npeers, uint64_t G,
                          const uint32_t *last_commit, const uint32_t *log_end,
                          const uint32_t *curr_term, const uint32_t *terms, uint32_t W,
                          uint32_t threshold, uint32_t *new_commit, int threads) {
#ifdef _OPENMP
    if (threads <= 0) threads = omp_get_max_threads();
#pragma omp parallel for schedule(static) num_threads(threads)
#endif
    for (uint64_t g = 0; g < G; g++) {
        uint32_t m[64];
        for (uint32_t q = 0; q < npeers && q < 64; q++) m[q] = match[(uint64_t)q * G + g];
        new_commit[g] = ssor_raft_scan(m, npeers, last_commit[g], log_end[g], curr_term[g],
                                       terms + g * (uint64_t)W, threshold);
    }
}

/* Incremental per-reply restatement of handle_msg_append_entries_reply for SUCCESSFUL replies of the current
 * term to a leader (raft/messages.rs:221-309 with conflict == None; check_term / heartbeat bookkeeping and the
 * conflict branch are outside the path).  State per group: next_slot / match_slot per peer ([P][G]), last_commit,
 * last_snap; the log is its term ring (term of slot s at terms[g*W + s % W]) and log_end.  threshold = quorum_cnt,
 * or CRaft's majority + fault_tolerance (craft/messages.rs:300-308). */
void ssor_raft_reply_stream(const uint32_t *rec_g, const uint8_t *rec_peer, const uint32_t *rec_end,
                            uint64_t n_rec, uint32_t npeers, uint32_t threshold, uint64_t G, uint32_t *next_slot,
                            uint32_t *match, uint32_t *last_commit, uint32_t *last_snap, const uint32_t *log_end,
                            const uint32_t *curr_term, const uint32_t *terms, uint32_t W) {
    for (uint64_t i = 0; i < n_rec; i++) {
        uint64_t g = rec_g[i];
        uint32_t peer = rec_peer[i], end_slot = rec_end[i];
        if (g >= G || peer >= npeers) continue;                     /* not a peer of this group */
        uint32_t *nx = &next_slot[(uint64_t)peer * G + g], *mt = &match[(uint64_t)peer * G + g];
        if (*nx > end_slot + 1) continue;                           /* :245-247 */
        *nx = end_slot + 1;                                         /* :248 */
        *mt = end_slot;                                             /* :252 */
        uint32_t new_commit = last_commit[g];                       /* :256-275 */
        for (uint32_t slot = last_commit[g] + 1; slot < log_end[g]; slot++) {
            if (terms[g * W + slot % W] != curr_term[g]) continue;
            uint32_t cnt = 1;
            for (uint32_t q = 0; q < npeers; q++) cnt += match[(uint64_t)q * G + g] >= slot ? 1u : 0u;
            if (cnt >= threshold) new_commit = slot;
        }
        last_commit[g] = new_commit;                                /* :295 */
        uint32_t snap0 = last_snap[g];                              /* :298-309 */
        for (uint32_t slot = snap0 + 1; slot <= end_slot; slot++) {
            uint32_t cnt = 1;
            for (uint32_t q = 0; q < npeers; q++) cnt += match[(uint64_t)q * G + g] >= slot ? 1u : 0u;
            if (cnt == npeers + 1) last_snap[g] = slot;
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * CRaft (craft/messages.rs:288-314, :677-690)
 * ------------------------------------------------------------------------------------------ */
uint32_t ssor_craft_threshold(uint32_t majority, uint32_t fault_tolerance, int full_copy_mode) {
    return full_copy_mode ? majority : majority + fault_tolerance;          /* :300-308 */
}

uint32_t ssor_craft_shadow_last_commit(const uint32_t *match, uint32_t npeers, uint32_t threshold) {
    /* :680-689: collect, sort_unstable, reverse, index [threshold - 2] */
    uint32_t v[64];
    if (npeers > 64 || threshold < 2 || threshold - 2 >= npeers) return 0;
    for (uint32_t i = 0; i < npeers; i++) v[i] = match[i];
    for (uint32_t i = 0; i < npeers; i++)
        for (uint32_t j = i + 1; j < npeers; j++)
            if (v[j] > v[i]) { uint32_t t = v[i]; v[i] = v[j]; v[j] = t; }
    return v[threshold - 2];
}

/* ------------------------------------------------------------------------------------------
 * Prepare-phase merge (rspaxos/messages.rs:182-259, crossword/messages.rs:233-312)
 * ------------------------------------------------------------------------------------------ */
void ssor_prepare_merge_stream(const uint8_t *has_vote, const uint64_t *bal, const uint32_t *mask,
                               uint32_t n_rep, uint64_t *max_bal, uint32_t *merged) {
    uint64_t prepare_max_bal = 0;     /* LeaderBookkeeping.prepare_max_bal starts at 0 */
    uint32_t cw = 0;                  /* shard set of inst.reqs_cw (null codeword) */
    for (uint32_t i = 0; i < n_rep; i++) {
        if (!has_vote[i]) continue;                      /* voted == None */
        if (bal[i] > prepare_max_bal) {                  /* discard current, take the replied codeword */
            prepare_max_bal = bal[i];
            cw = mask[i];
        } else if (bal[i] == prepare_max_bal) {          /* absorb_other: takes shards not yet held */
            cw |= mask[i];
        }
    }
    *max_bal = prepare_max_bal;
    *merged = cw;
}

uint32_t ssor_prepare_decide(uint32_t merged, uint32_t acks_cnt, uint32_t data_shards, uint32_t population,
                             uint32_t fault_tolerance) {
    uint32_t avail = popc32(merged);
    uint32_t avail_data = popc32(merged & ((data_shards >= 32) ? 0xffffffffu : ((1u << data_shards) - 1u)));
    uint32_t act;
    if (avail >= data_shards) {
        act = SSOR_PM_USE;
        if (avail_data < data_shards) act |= SSOR_PM_RECONSTRUCT;
    } else if (acks_cnt >= population - fault_tolerance) {
        act = SSOR_PM_NULL;
        avail = data_shards;          /* from_data(empty batch): all d data shards present, no parity */
    } else {
        return 0;                     /* "not yet for this instance" */
    }
    if (avail < population) act |= SSOR_PM_PARITY;
    return act;
}

/* crossword/gossiping.rs:35-84 */
uint32_t ssor_gossip_targets_excl(uint32_t me, uint32_t population, uint32_t data_shards, uint32_t src_peer,
                                  uint32_t avail, const uint32_t *assignment, uint32_t peer_alive, uint32_t *excl) {
    uint32_t targets = 0;
    for (uint32_t pp = me + 1; pp < me + population; pp++) {          /* :54 */
        uint32_t peer = pp % population;
        if (peer == src_peer) continue;                               /* :56-59 */
        if (!((peer_alive >> peer) & 1u)) continue;                   /* :60-63 */
        uint32_t useful = assignment[peer] & ~avail;                  /* :67-72 */
        if (useful != 0) {
            excl[peer] = avail;                                       /* :74 (clone before marking) */
            targets |= 1u << peer;
            avail |= useful;                                          /* :75-77 */
        }
        if (popc32(avail) >= data_shards) break;                      /* :80-82 */
    }
    return targets;
}
