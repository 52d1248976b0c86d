// summerset_host.hpp -- header-only C++17 host side above the C ABI (include/summerset_b200.h).
//
// The reference's host code for this path is Rust; no Rust toolchain exists in the build image, so the
// host-side mirror is C++ with the reference's names, argument meaning and error behaviour:
//   ssb::Bitmap        <- src/utils/bitmap.rs            (u8 id -> bool bitset)
//   ssb::ReedSolomon   <- reed_solomon_erasure::galois_8::ReedSolomon as used by src/utils/rscoding.rs
//   ssb::RSCodeword    <- src/utils/rscoding.rs          (T = an already serialised byte string)
//   ssb::Acceptor      <- the follower side of rspaxos/messages.rs handle_msg_accept + durability.rs's AcceptReply,
//                         batched over many groups (ss_acceptor_*, device buffers)
// Only bookkeeping happens here.  Every shard byte is computed by the CUDA kernels behind the C ABI;
// a failing ABI call becomes a SummersetError (src/utils/error.rs:6-14) -- there is no CPU fallback.
#pragma once
#include <cstdint>
#include <cstring>
#include <optional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/summerset_b200.h"

namespace ssb {

struct SummersetError : std::runtime_error {
    int code;
    SummersetError(int c, const std::string &m) : std::runtime_error(m), code(c) {}
    static SummersetError msg(const std::string &m) { return SummersetError(SS_ERR_INVALID_ARG, m); }
};

inline void check(int rc) {
    if (rc != SS_OK) throw SummersetError(rc, ss_last_error());
}

// ---------------------------------------------------------------------------------------------
// Bitmap (src/utils/bitmap.rs:17-149)
// ---------------------------------------------------------------------------------------------
class Bitmap {
  public:
    Bitmap(uint8_t size, bool ones) : size_(size), words_((size + 63u) / 64u, 0) {
        if (size == 0) throw std::logic_error("invalid bitmap size 0");   // bitmap.rs:64 (panic)
        if (ones)
            for (unsigned i = 0; i < size; ++i) words_[i / 64] |= 1ull << (i % 64);
    }
    static Bitmap from(uint8_t size, const std::vector<uint8_t> &ones) {       // bitmap.rs:151-185
        Bitmap b(size, false);
        for (uint8_t i : ones) b.set(i, true);
        return b;
    }
    void set(uint8_t idx, bool flag) {                                         // bitmap.rs:74-84
        if (idx >= size_) throw SummersetError(SS_ERR_INVALID_INDEX, "index " + std::to_string(idx) + " out of bound");
        if (flag) words_[idx / 64] |= 1ull << (idx % 64);
        else words_[idx / 64] &= ~(1ull << (idx % 64));
    }
    bool get(uint8_t idx) const {                                              // bitmap.rs:87-97
        if (idx >= size_) throw SummersetError(SS_ERR_INVALID_INDEX, "index " + std::to_string(idx) + " out of bound");
        return (words_[idx / 64] >> (idx % 64)) & 1ull;
    }
    uint8_t size() const { return size_; }
    uint8_t count() const {                                                    // bitmap.rs:111-113
        unsigned c = 0;
        for (uint64_t w : words_) c += static_cast<unsigned>(__builtin_popcountll(w));
        return static_cast<uint8_t>(c);
    }
    void flip() {                                                              // bitmap.rs:117-119
        for (unsigned i = 0; i < size_; ++i) words_[i / 64] ^= 1ull << (i % 64);
    }
    void union_with(const Bitmap &o) {                                         // bitmap.rs:123-135
        if (size_ != o.size_)
            throw SummersetError::msg("unioning sizes mismatch: " + std::to_string(size_) + " != " + std::to_string(o.size_));
        for (size_t i = 0; i < words_.size(); ++i) words_[i] |= o.words_[i];
    }
    void clear() { std::fill(words_.begin(), words_.end(), 0ull); }
    std::vector<uint8_t> to_vec() const {                                      // bitmap.rs:211-229
        std::vector<uint8_t> v;
        for (unsigned i = 0; i < size_; ++i)
            if (get(static_cast<uint8_t>(i))) v.push_back(static_cast<uint8_t>(i));
        return v;
    }
    uint64_t mask() const { return words_[0]; }                                // ids < 64: the device-side vote mask
    bool operator==(const Bitmap &o) const { return size_ == o.size_ && words_ == o.words_; }

  private:
    uint8_t size_;
    std::vector<uint64_t> words_;
};

// ---------------------------------------------------------------------------------------------
// ReedSolomon: RAII over ss_ctx + ss_rs_coder
// ---------------------------------------------------------------------------------------------
class ReedSolomon {
  public:
    ReedSolomon(size_t data_shards, size_t parity_shards, int device = 0) {
        check(ss_ctx_create(device, &ctx_));
        int rc = ss_rs_coder_create(ctx_, static_cast<int>(data_shards), static_cast<int>(parity_shards), &coder_);
        if (rc != SS_OK) {
            std::string m = ss_last_error();
            ss_ctx_destroy(ctx_);
            throw SummersetError(rc, m);
        }
    }
    ~ReedSolomon() {
        ss_rs_coder_destroy(coder_);
        ss_ctx_destroy(ctx_);
    }
    ReedSolomon(const ReedSolomon &) = delete;
    ReedSolomon &operator=(const ReedSolomon &) = delete;

    size_t data_shard_count() const { return static_cast<size_t>(ss_rs_data_shard_count(coder_)); }
    size_t parity_shard_count() const { return static_cast<size_t>(ss_rs_parity_shard_count(coder_)); }
    size_t total_shard_count() const { return static_cast<size_t>(ss_rs_total_shard_count(coder_)); }

    // rs.encode(slices): all d+p shards, parity overwritten
    void encode(std::vector<std::vector<uint8_t>> &shards) const {
        const size_t len = shards.empty() ? 0 : shards[0].size();
        for (auto &s : shards)
            if (s.size() != len) throw SummersetError(SS_ERR_INCORRECT_SHARD_SIZE, "incorrect shard size");
        std::vector<uint8_t *> p;
        for (auto &s : shards) p.push_back(s.data());
        check(ss_rs_encode(coder_, p.data(), p.size(), len));
    }
    void reconstruct(std::vector<std::optional<std::vector<uint8_t>>> &shards) const { recon(shards, false); }
    void reconstruct_data(std::vector<std::optional<std::vector<uint8_t>>> &shards) const { recon(shards, true); }
    bool verify(const std::vector<std::vector<uint8_t>> &shards) const {
        const size_t len = shards.empty() ? 0 : shards[0].size();
        std::vector<const uint8_t *> p;
        for (auto &s : shards) p.push_back(s.data());
        int ok = 0;
        check(ss_rs_verify(coder_, p.data(), p.size(), len, &ok));
        return ok != 0;
    }
    ss_rs_coder *handle() const { return coder_; }
    ss_ctx *context() const { return ctx_; }

  private:
    void recon(std::vector<std::optional<std::vector<uint8_t>>> &shards, bool data_only) const {
        size_t len = 0;
        for (auto &s : shards)
            if (s) { len = s->size(); break; }
        std::vector<uint8_t> present(shards.size());
        std::vector<std::vector<uint8_t>> tmp(shards.size());
        std::vector<uint8_t *> p(shards.size());
        for (size_t i = 0; i < shards.size(); ++i) {
            present[i] = shards[i] ? 1 : 0;
            if (shards[i]) p[i] = shards[i]->data();
            else { tmp[i].assign(len ? len : 1, 0); p[i] = tmp[i].data(); }
        }
        check(data_only ? ss_rs_reconstruct_data(coder_, p.data(), present.data(), p.size(), len)
                        : ss_rs_reconstruct(coder_, p.data(), present.data(), p.size(), len));
        for (size_t i = 0; i < shards.size(); ++i)
            if (!shards[i] && present[i]) shards[i] = std::move(tmp[i]);
    }
    ss_ctx *ctx_ = nullptr;
    ss_rs_coder *coder_ = nullptr;
};

// ---------------------------------------------------------------------------------------------
// RSCodeword (src/utils/rscoding.rs:15-606), T = serialized bytes
// ---------------------------------------------------------------------------------------------
class RSCodeword {
  public:
    using Bytes = std::vector<uint8_t>;

    static RSCodeword from_data(const Bytes &data, uint8_t d, uint8_t p) {    // rscoding.rs:223-243
        return internal_new(data, &data, data.size(), d, p);
    }
    static RSCodeword from_null(uint8_t d, uint8_t p) {                       // rscoding.rs:246-251
        return internal_new(std::nullopt, nullptr, 0, d, p);
    }

    RSCodeword subset_copy(const Bitmap &subset, bool copy_data) const {      // rscoding.rs:255-293
        if (data_len_ == 0) throw SummersetError::msg("codeword is null");
        RSCodeword out(*this);
        for (auto &s : out.shards) s.reset();
        for (unsigned i = 0; i < subset.size(); ++i) {
            if (!subset.get(static_cast<uint8_t>(i))) continue;
            if (i >= shards.size()) throw SummersetError::msg("shard index " + std::to_string(i) + " out-of-bound");
            out.shards[i] = shards[i];
        }
        if (!copy_data) out.data_copy.reset();
        return out;
    }

    void absorb_other(RSCodeword other) {                                     // rscoding.rs:296-345
        if (d_ != other.d_) throw SummersetError::msg("num_data_shards mismatch");
        if (p_ != other.p_) throw SummersetError::msg("num_parity_shards mismatch");
        if (data_len_ != 0 && data_len_ != other.data_len_) throw SummersetError::msg("data_len mismatch");
        if (shard_len_ != 0 && shard_len_ != other.shard_len_) throw SummersetError::msg("shard_len mismatch");
        if (data_len_ == 0) { data_len_ = other.data_len_; shard_len_ = other.shard_len_; }
        for (size_t i = 0; i < other.shards.size(); ++i)
            if (other.shards[i] && !shards[i]) shards[i] = std::move(other.shards[i]);
    }

    uint8_t num_data_shards() const { return d_; }
    uint8_t num_parity_shards() const { return p_; }
    uint8_t num_shards() const { return static_cast<uint8_t>(shards.size()); }
    uint8_t avail_data_shards() const { return count(0, d_); }
    uint8_t avail_parity_shards() const { return count(d_, shards.size()); }
    uint8_t avail_shards() const { return count(0, shards.size()); }
    Bitmap avail_shards_map() const {                                         // rscoding.rs:400-408
        Bitmap m(num_shards(), false);
        for (size_t i = 0; i < shards.size(); ++i)
            if (shards[i]) m.set(static_cast<uint8_t>(i), true);
        return m;
    }
    size_t data_len() const { return data_len_; }
    size_t shard_len() const { return shard_len_; }

    void compute_parity(const ReedSolomon *rs) {                              // rscoding.rs:447-486
        if (data_len_ == 0) throw SummersetError::msg("codeword is null");
        if (p_ == 0) return;
        if (!rs) throw SummersetError::msg("ReedSolomon coder is None");
        splits_match(*rs);
        if (avail_data_shards() < d_) throw SummersetError::msg("not all data shards present");
        std::vector<Bytes> all;
        for (size_t i = 0; i < shards.size(); ++i) all.push_back(shards[i] ? *shards[i] : Bytes(shard_len_, 0));
        rs->encode(all);
        for (size_t i = 0; i < shards.size(); ++i) shards[i] = std::move(all[i]);
    }
    void reconstruct_all(const ReedSolomon *rs) { reconstruct(rs, false); }   // rscoding.rs:524-529
    void reconstruct_data(const ReedSolomon *rs) { reconstruct(rs, true); }   // rscoding.rs:532-537

    bool verify_parity(const ReedSolomon *rs) {                               // rscoding.rs:542-576
        if (data_len_ == 0) throw SummersetError::msg("codeword is null");
        if (p_ == 0) {
            if (avail_data_shards() == d_) return true;
            throw SummersetError::msg("not all shards present");
        }
        if (!rs) throw SummersetError::msg("ReedSolomon is None");
        splits_match(*rs);
        if (avail_shards() < num_shards()) throw SummersetError::msg("not all shards present");
        std::vector<Bytes> all;
        for (auto &s : shards) all.push_back(*s);
        return rs->verify(all);
    }

    const Bytes &get_data() {                                                 // rscoding.rs:581-606
        if (data_len_ == 0) throw SummersetError::msg("codeword is null");
        if (avail_data_shards() < d_) throw SummersetError::msg("not all data shards present");
        if (!data_copy) {                                                      // ShardsReader, rscoding.rs:649-682
            Bytes cat;
            for (unsigned i = 0; i < d_; ++i) cat.insert(cat.end(), shards[i]->begin(), shards[i]->end());
            cat.resize(data_len_);
            data_copy = std::move(cat);
        }
        return *data_copy;
    }

    std::vector<std::optional<Bytes>> shards;
    std::optional<Bytes> data_copy;

  private:
    static RSCodeword internal_new(std::optional<Bytes> copy, const Bytes *bytes, size_t data_len, uint8_t d,
                                   uint8_t p) {                               // rscoding.rs:165-220
        if (d == 0) throw SummersetError::msg("num_data_shards is zero");
        RSCodeword cw;
        cw.d_ = d; cw.p_ = p; cw.data_len_ = data_len;
        cw.shard_len_ = (data_len % d == 0) ? data_len / d : data_len / d + 1;
        cw.shards.resize(size_t(d) + p);
        if (bytes) {
            Bytes padded(*bytes);
            padded.resize(cw.shard_len_ * d, 0);
            for (unsigned i = 0; i < d; ++i)
                cw.shards[i] = Bytes(padded.begin() + long(i * cw.shard_len_), padded.begin() + long((i + 1) * cw.shard_len_));
        }
        cw.data_copy = std::move(copy);
        return cw;
    }
    uint8_t count(size_t a, size_t b) const {
        unsigned c = 0;
        for (size_t i = a; i < b; ++i) c += shards[i] ? 1u : 0u;
        return static_cast<uint8_t>(c);
    }
    void splits_match(const ReedSolomon &rs) const {                          // rscoding.rs:424-443
        if (rs.data_shard_count() != d_) throw SummersetError::msg("num_data_shards mismatch");
        if (rs.parity_shard_count() != p_) throw SummersetError::msg("num_parity_shards mismatch");
    }
    void reconstruct(const ReedSolomon *rs, bool data_only) {                 // rscoding.rs:490-520
        if (data_len_ == 0) throw SummersetError::msg("codeword is null");
        if (p_ == 0) {
            if (avail_data_shards() == d_) return;
            throw SummersetError::msg("insufficient data shards");
        }
        if (!rs) throw SummersetError::msg("ReedSolomon coder is None");
        splits_match(*rs);
        if (data_only) rs->reconstruct_data(shards);
        else rs->reconstruct(shards);
    }
    uint8_t d_ = 0, p_ = 0;
    size_t data_len_ = 0, shard_len_ = 0;
};

// ---------------------------------------------------------------------------------------------
// Acceptor: RAII over ss_acceptor (follower side of the RSPaxos / Crossword accept path).  handle_msg_accept runs for a
// whole batch of received Accept frames; the AcceptData records it returns are what the host appends to its WAL, and
// the AcceptReply cells go out (send_msg to reply_dst[i]) only once those records are durable.
// ---------------------------------------------------------------------------------------------
class Acceptor {
  public:
    Acceptor(ss_ctx *ctx, const ss_acceptor_config &cfg, uint64_t n_groups) { check(ss_acceptor_create(ctx, &cfg, n_groups, &acc_)); }
    ~Acceptor() { ss_acceptor_destroy(acc_); }
    Acceptor(const Acceptor &) = delete;
    Acceptor &operator=(const Acceptor &) = delete;

    // every pointer is a device pointer; see ss_acceptor_accept for the outputs
    void handle_msg_accept(const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                           const uint8_t *frame_peer, uint64_t n_frames, uint8_t *store, uint64_t store_capacity,
                           uint64_t *store_off, uint8_t *wal, uint64_t wal_capacity, uint64_t *wal_off, uint32_t *wal_len,
                           uint8_t *replies, uint32_t *reply_len, uint8_t *reply_dst, uint32_t *verdict, uint64_t *totals) {
        check(ss_acceptor_accept(acc_, buf, buf_len, frame_off, frame_group, frame_peer, n_frames, store, store_capacity, store_off,
                                 wal, wal_capacity, wal_off, wal_len, replies, reply_len, reply_dst, verdict, totals));
    }
    // start_slot moves to upto[g] (device [G]), at most 64 slots at a time
    void advance_start_slot(const uint64_t *upto) { check(ss_acceptor_advance(acc_, upto)); }
    // heard_heartbeat's commit walk; newly[g] (may be NULL) = the instances to log as CommitSlot (ss_wal_commit_pack_dev)
    void heard_heartbeat(const uint32_t *group, const uint8_t *peer, const uint64_t *ballot, const uint64_t *commit_bar,
                         const uint64_t *exec_bar, uint64_t n_records, uint64_t *newly) {
        check(ss_acceptor_heartbeat(acc_, group, peer, ballot, commit_bar, exec_bar, n_records, newly));
    }
    // once those CommitSlot records are durable: handle_logged_commit_slot's walk, request batches into out
    void execute(uint8_t *out, uint64_t out_capacity, uint32_t *rec_group, uint64_t *rec_slot, uint64_t *rec_off, uint32_t *rec_len,
                 uint64_t rec_capacity, uint64_t *totals) {
        check(ss_acceptor_execute(acc_, out, out_capacity, rec_group, rec_slot, rec_off, rec_len, rec_capacity, totals));
    }
    // handle_msg_reconstruct: Reconstruct frames (PeerMsg variant 4) in, ReconstructReply frames (variant 5) into out;
    // reply i goes to frame_peer[i]
    void reconstruct_serve(const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                           const uint8_t *frame_peer, uint64_t n_frames, uint8_t *out, uint64_t out_capacity, uint64_t *reply_off,
                           uint64_t *reply_len, uint32_t *verdict, uint64_t *total, uint32_t reconstruct_variant = 4,
                           uint32_t reply_variant = 5) {
        check(ss_acceptor_reconstruct_serve(acc_, buf, buf_len, frame_off, frame_group, frame_peer, n_frames, reconstruct_variant,
                                            reply_variant, out, out_capacity, reply_off, reply_len, verdict, total));
    }
    // handle_msg_reconstruct_reply: the shards of ReconstructReply frames into new regions of store; execute() then runs
    // what now holds d shards
    void absorb(const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group, const uint8_t *frame_peer,
                uint64_t n_frames, uint8_t *store, uint64_t store_capacity, uint32_t *absorbed, uint32_t *verdict, uint64_t *total,
                uint32_t reply_variant = 5) {
        check(ss_acceptor_absorb(acc_, buf, buf_len, frame_off, frame_group, frame_peer, n_frames, reply_variant, store, store_capacity,
                                 absorbed, verdict, total));
    }
    // handle_msg_prepare: Prepare frames (PeerMsg variant 0) in, one 32-byte WalEntry::PrepareBal cell (variant 0) per
    // covered slot out; a capacity cut leaves a prefix of the frames applied (see the header)
    void prepare(const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group, const uint8_t *frame_peer,
                 uint64_t n_frames, uint8_t *wal, uint64_t wal_capacity, uint32_t *rec_group, uint64_t *rec_slot, uint32_t *rec_frame,
                 uint64_t rec_capacity, uint32_t *verdict, uint64_t *totals, uint32_t prepare_variant = 0, uint32_t wal_variant = 0) {
        check(ss_acceptor_prepare(acc_, buf, buf_len, frame_off, frame_group, frame_peer, n_frames, prepare_variant, wal_variant, wal,
                                  wal_capacity, rec_group, rec_slot, rec_frame, rec_capacity, verdict, totals));
    }
    // once those PrepareBal records are durable: PrepareReply frames (variant 1) into out; reply k goes to reply_dst[k]
    void prepare_reply(const uint32_t *rec_group, const uint64_t *rec_slot, uint64_t n_records, uint8_t *out, uint64_t out_capacity,
                       uint64_t *reply_off, uint64_t *reply_len, uint8_t *reply_dst, uint64_t *total, uint32_t reply_variant = 1) {
        check(ss_acceptor_prepare_reply(acc_, rec_group, rec_slot, n_records, reply_variant, out, out_capacity, reply_off, reply_len,
                                        reply_dst, total));
    }
    // recover_apply_entry over a group-tagged batch of WAL records (PrepareBal variant 0, AcceptData cfg.wal_variant,
    // CommitSlot variant 2), each group's in WAL order; the defining shards go to store.  A group cut by the window or the
    // store is finished by re-submitting its unapplied records (see the header)
    void recover(const uint8_t *buf, uint64_t buf_len, const uint64_t *rec_off, const uint32_t *rec_group, uint64_t n_records,
                 uint8_t *store, uint64_t store_capacity, uint32_t *verdict, uint64_t *total, uint32_t prepare_variant = 0,
                 uint32_t commit_variant = 2) {
        check(ss_acceptor_recover(acc_, buf, buf_len, rec_off, rec_group, n_records, prepare_variant, commit_variant, store,
                                  store_capacity, verdict, total));
    }
    // Crossword trigger_gossiping over the listed groups (NULL: all; leave out the groups this replica leads):
    // Reconstruct frames (variant 4) for peer frame_dst[f]; a capacity cut leaves a prefix of the groups written
    void gossip(const uint32_t *groups, uint64_t n_listed, const uint32_t *peer_alive, uint64_t tail_ignores, uint64_t batch_size,
                uint8_t *out, uint64_t out_capacity, uint32_t *frame_group, uint8_t *frame_dst, uint64_t *frame_off, uint32_t *frame_len,
                uint64_t frame_capacity, uint64_t *totals, uint32_t reconstruct_variant = 4) {
        check(ss_acceptor_gossip(acc_, groups, n_listed, peer_alive, tail_ignores, batch_size, reconstruct_variant, out, out_capacity,
                                 frame_group, frame_dst, frame_off, frame_len, frame_capacity, totals));
    }
    // become_a_leader's reconstruct reads: Reconstruct frames (variant 4) to broadcast, chunk_size = msg_chunk_size
    void step_up_reads(const uint32_t *groups, uint64_t n_listed, uint64_t chunk_size, uint8_t *out, uint64_t out_capacity,
                       uint32_t *frame_group, uint8_t *frame_dst, uint64_t *frame_off, uint32_t *frame_len, uint64_t frame_capacity,
                       uint64_t *totals, uint32_t reconstruct_variant = 4) {
        check(ss_acceptor_step_up_reads(acc_, groups, n_listed, chunk_size, reconstruct_variant, out, out_capacity, frame_group, frame_dst,
                                        frame_off, frame_len, frame_capacity, totals));
    }
    // become_a_leader's Prepare half: a greater ballot, the in-progress instances Preparing with source = me, 32-byte
    // PrepareBal cells (variant 0) and one 32-byte Prepare frame (variant 0) per group to broadcast; once the records are
    // durable, prepare_reply() on them gives the leader's own votes (reply_dst = me).  A capacity cut leaves a prefix of
    // the groups applied (see the header)
    void step_up(const uint32_t *groups, uint64_t n_listed, uint8_t *wal, uint64_t wal_capacity, uint32_t *rec_group, uint64_t *rec_slot,
                 uint64_t rec_capacity, uint8_t *out, uint64_t out_capacity, uint32_t *frame_group, uint8_t *frame_dst, uint64_t *frame_off,
                 uint32_t *frame_len, uint64_t frame_capacity, uint32_t *verdict, uint64_t *ballot, uint64_t *trigger_slot,
                 uint64_t *endprep_slot, uint64_t *totals, uint32_t prepare_variant = 0, uint32_t wal_variant = 0) {
        check(ss_acceptor_step_up(acc_, groups, n_listed, prepare_variant, wal_variant, wal, wal_capacity, rec_group, rec_slot,
                                  rec_capacity, out, out_capacity, frame_group, frame_dst, frame_off, frame_len, frame_capacity, verdict,
                                  ballot, trigger_slot, endprep_slot, totals));
    }
    ss_acceptor_gossip_view gossip_view() const {
        ss_acceptor_gossip_view v;
        check(ss_acceptor_gossip_view_get(acc_, &v));
        return v;
    }
    ss_acceptor_view view() const {
        ss_acceptor_view v;
        check(ss_acceptor_view_get(acc_, &v));
        return v;
    }
    ss_acceptor_commit_view commit_view() const {
        ss_acceptor_commit_view v;
        check(ss_acceptor_commit_view_get(acc_, &v));
        return v;
    }
    ss_acceptor_prepare_view prepare_view() const {
        ss_acceptor_prepare_view v;
        check(ss_acceptor_prepare_view_get(acc_, &v));
        return v;
    }
    ss_acceptor *handle() const { return acc_; }

  private:
    ss_acceptor *acc_ = nullptr;
};

// the CRaft follower (ss_follower_*): AppendEntries frames in, LogEntry / Metadata records and AppendEntriesReply cells out
class Follower {
  public:
    Follower(ss_ctx *ctx, const ss_follower_config &cfg, uint64_t n_groups) { check(ss_follower_create(ctx, &cfg, n_groups, &fol_)); }
    ~Follower() { ss_follower_destroy(fol_); }
    Follower(const Follower &) = delete;
    Follower &operator=(const Follower &) = delete;

    // every pointer is a device pointer; see ss_follower_append for the outputs
    void handle_msg_append_entries(const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                                   const uint8_t *frame_peer, uint64_t n_frames, uint8_t *store, uint64_t store_capacity,
                                   uint64_t *store_off, uint8_t *wal, uint64_t wal_capacity, uint64_t *wal_off, uint64_t *wal_len,
                                   uint8_t *meta, uint32_t *meta_len, uint8_t *replies, uint32_t *reply_len, uint8_t *reply_dst,
                                   uint64_t *trunc_slot, uint32_t *verdict, uint64_t *commit_lo, uint64_t *totals) {
        check(ss_follower_append(fol_, buf, buf_len, frame_off, frame_group, frame_peer, n_frames, store, store_capacity, store_off,
                                 wal, wal_capacity, wal_off, wal_len, meta, meta_len, replies, reply_len, reply_dst, trunc_slot,
                                 verdict, commit_lo, totals));
    }
    // the snapshot's start_slot move, never past last_commit
    void advance_start_slot(const uint64_t *upto) { check(ss_follower_advance(fol_, upto)); }
    ss_follower_view view() const {
        ss_follower_view v{};
        check(ss_follower_view_get(fol_, &v));
        return v;
    }
    ss_follower_exec_view exec_view() const {
        ss_follower_exec_view v{};
        check(ss_follower_exec_view_get(fol_, &v));
        return v;
    }
    // the committed entries' request batches (see ss_follower_execute); pass last_exec to advance_start_slot
    void execute(uint8_t *out, uint64_t out_capacity, uint32_t *rec_group, uint64_t *rec_slot, uint64_t *rec_off, uint32_t *rec_len,
                 uint64_t rec_capacity, uint64_t *totals = nullptr) {
        check(ss_follower_execute(fol_, out, out_capacity, rec_group, rec_slot, rec_off, rec_len, rec_capacity, totals));
    }
    // a new leader's Reconstruct frames answered from the held shards (see ss_follower_reconstruct_serve)
    void handle_msg_reconstruct(const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                                const uint8_t *frame_peer, uint64_t n_frames, uint8_t *out, uint64_t out_capacity, uint64_t *reply_off,
                                uint64_t *reply_len, uint32_t *verdict, uint64_t *total = nullptr, uint32_t reconstruct_variant = 4,
                                uint32_t reply_variant = 5) {
        check(ss_follower_reconstruct_serve(fol_, buf, buf_len, frame_off, frame_group, frame_peer, n_frames, reconstruct_variant,
                                            reply_variant, out, out_capacity, reply_off, reply_len, verdict, total));
    }
    // elections: the state beside the follower's, allocated on first use (see ss_follower_vote_view)
    ss_follower_vote_view vote_view() const {
        ss_follower_vote_view v{};
        check(ss_follower_vote_view_get(fol_, &v));
        return v;
    }
    // become_a_candidate for the listed groups: Metadata cells, then RequestVote frames to broadcast (see ss_follower_campaign)
    void become_a_candidate(const uint32_t *groups, uint64_t n_listed, const uint8_t *timeout_source, uint8_t *meta, uint32_t *meta_len,
                            uint8_t *frames, uint32_t *frame_len, uint8_t *frame_dst, uint32_t *verdict, uint32_t request_vote_variant = 2) {
        check(ss_follower_campaign(fol_, groups, n_listed, timeout_source, request_vote_variant, meta, meta_len, frames, frame_len, frame_dst,
                                   verdict));
    }
    // RequestVote frames answered (see ss_follower_vote)
    void handle_msg_request_vote(const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                                 const uint8_t *frame_peer, uint64_t n_frames, uint8_t *meta, uint32_t *meta_len, uint8_t *replies,
                                 uint32_t *reply_len, uint8_t *reply_dst, uint32_t *verdict, uint32_t request_vote_variant = 2,
                                 uint32_t reply_variant = 3) {
        check(ss_follower_vote(fol_, buf, buf_len, frame_off, frame_group, frame_peer, n_frames, request_vote_variant, reply_variant, meta,
                               meta_len, replies, reply_len, reply_dst, verdict));
    }
    // RequestVoteReply frames tallied; won_group / won_term ([n_groups]) go to craft_step_up (see ss_follower_tally)
    void handle_msg_request_vote_reply(const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                                       const uint8_t *frame_peer, uint64_t n_frames, uint8_t *meta, uint32_t *meta_len, uint32_t *verdict,
                                       uint32_t *won_group, uint64_t *won_term, uint64_t *n_won = nullptr, uint32_t reply_variant = 3) {
        check(ss_follower_tally(fol_, buf, buf_len, frame_off, frame_group, frame_peer, n_frames, reply_variant, meta, meta_len, verdict,
                                won_group, won_term, n_won));
    }
    // recover_from_wal over a group-tagged batch of Metadata (cfg.meta_variant) and LogEntry (cfg.log_variant) records,
    // each group's Metadata first and the rest in WAL order; the shards go to store.  A group cut by the store is
    // finished by re-submitting its STORE_FULL records (see ss_follower_recover)
    void recover(const uint8_t *buf, uint64_t buf_len, const uint64_t *rec_off, const uint32_t *rec_group, uint64_t n_records,
                 uint8_t *store, uint64_t store_capacity, uint32_t *verdict, uint64_t *total = nullptr) {
        check(ss_follower_recover(fol_, buf, buf_len, rec_off, rec_group, n_records, store, store_capacity, verdict, total));
    }
    // the handle, for ss_engine_craft_step_up
    const ss_follower *get() const { return fol_; }

  private:
    ss_follower *fol_ = nullptr;
};

// the leader's side: AppendEntriesReply frames -> the records ss_engine_raft_ingest takes (rec_group UINT32_MAX: dropped)
inline void append_reply_parse(ss_ctx *ctx, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                               const uint8_t *frame_peer, const uint32_t *curr_term, uint64_t n_frames, uint64_t n_groups,
                               uint32_t *rec_group, uint8_t *rec_peer, uint32_t *rec_end_slot, uint64_t *rec_term,
                               uint64_t *rec_conflict_term, uint64_t *rec_conflict_slot, uint32_t *rec_kind, uint32_t reply_variant = 1) {
    check(ss_append_reply_parse_dev(ctx, buf, buf_len, frame_off, frame_group, frame_peer, curr_term, n_frames, n_groups, reply_variant,
                                    rec_group, rec_peer, rec_end_slot, rec_term, rec_conflict_term, rec_conflict_slot, rec_kind));
}

// the CRaft leader's log on a CRaft engine; every pointer is a device pointer (see the header's ss_engine_craft_* block)
inline ss_engine_craft_log_view craft_log_view(ss_engine *e) {
    ss_engine_craft_log_view v{};
    check(ss_engine_craft_log_view_get(e, &v));
    return v;
}
inline void craft_propose(ss_engine *e, uint32_t me, const uint8_t *arena, const uint64_t *data_off, const uint32_t *data_len,
                          uint8_t *shards, uint64_t plane_stride, uint64_t *shard_off, uint64_t *slot_out, uint8_t *wal,
                          uint64_t wal_capacity, uint64_t *wal_off, uint64_t *wal_len, const uint64_t *log_offset = nullptr,
                          uint64_t *need = nullptr, bool full_copy = false) {
    check(ss_engine_craft_propose(e, me, arena, data_off, data_len, shards, plane_stride, shard_off, slot_out, need, log_offset, wal,
                                  wal_capacity, wal_off, wal_len, full_copy ? 1 : 0));
}
inline void append_pack(ss_engine *e, const ss_append_pack_spec &spec, const uint64_t *want_end, uint8_t *out, uint64_t out_capacity,
                        uint64_t *frame_off, uint64_t *frame_len, uint32_t *frame_group, uint8_t *frame_peer, uint64_t max_frames,
                        uint64_t *n_frames, uint32_t *pair_status, uint64_t *total = nullptr) {
    check(ss_frame_append_pack_dev(e, &spec, want_end, out, out_capacity, frame_off, frame_len, frame_group, frame_peer, max_frames,
                                   n_frames, pair_status, total));
}
inline void craft_backoff(ss_engine *e, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                          const uint8_t *frame_peer, const uint32_t *rec_kind, uint64_t n_frames, uint64_t *want_end,
                          uint32_t reply_variant = 1) {
    check(ss_engine_craft_backoff(e, buf, buf_len, frame_off, frame_group, frame_peer, rec_kind, n_frames, reply_variant, want_end));
}
inline void craft_advance(ss_engine *e, const uint64_t *upto) { check(ss_engine_craft_advance(e, upto)); }
inline void craft_set_full_copy(ss_engine *e, bool full_copy) { check(ss_engine_craft_set_full_copy(e, full_copy ? 1 : 0)); }
inline ss_engine_craft_exec_view craft_exec_view(ss_engine *e) {
    ss_engine_craft_exec_view v{};
    check(ss_engine_craft_exec_view_get(e, &v));
    return v;
}
inline void craft_execute(ss_engine *e, uint8_t *out, uint64_t out_capacity, uint32_t *rec_group, uint64_t *rec_slot, uint64_t *rec_off,
                          uint32_t *rec_len, uint64_t rec_capacity, uint64_t *totals = nullptr) {
    check(ss_engine_craft_execute(e, out, out_capacity, rec_group, rec_slot, rec_off, rec_len, rec_capacity, totals));
}
// fail-over: step-up from this replica's follower, the Reconstruct reads, the replies absorbed (ss_engine_craft_step_up ...)
inline ss_engine_craft_recon_view craft_recon_view(ss_engine *e) {
    ss_engine_craft_recon_view v{};
    check(ss_engine_craft_recon_view_get(e, &v));
    return v;
}
inline void craft_step_up(ss_engine *e, const Follower &follower, const uint32_t *groups, uint64_t n_listed, const uint64_t *term,
                          uint8_t *shards, uint64_t plane_stride, uint64_t *shard_off, uint32_t *verdict, uint64_t *need = nullptr) {
    check(ss_engine_craft_step_up(e, follower.get(), groups, n_listed, term, shards, plane_stride, shard_off, need, verdict));
}
// RSPaxos / Crossword fail-over on the new leader: PrepareReply frames (its own and its peers') absorbed after
// Acceptor::step_up; the decided list feeds ss_frame_accept_pack_ragged_dev, and the leader's own frame goes to its own
// Acceptor::accept in the same turn (see ss_engine_prepare_absorb for the capacity cut and the host's part)
inline void prepare_absorb(ss_engine *e, Acceptor &acceptor, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off,
                           const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames, const uint64_t *bal_prep_sent,
                           const uint8_t *policy, uint8_t *shards, uint64_t plane_stride, uint64_t *store_used, uint8_t *wal,
                           uint64_t wal_capacity, uint32_t *rec_group, uint64_t *rec_slot, uint64_t rec_capacity, uint64_t *dec_slot,
                           uint64_t *dec_ballot, uint64_t *dec_shard_off, uint32_t *dec_data_len, uint8_t *dec_policy,
                           uint32_t *dec_group, uint64_t dec_capacity, uint64_t *pending, uint32_t *verdict,
                           uint64_t *totals = nullptr, uint32_t reply_variant = 1, uint32_t wal_variant = 0) {
    check(ss_engine_prepare_absorb(e, acceptor.handle(), buf, buf_len, frame_off, frame_group, frame_peer, n_frames, reply_variant,
                                   wal_variant, bal_prep_sent, policy, shards, plane_stride, store_used, wal, wal_capacity, rec_group,
                                   rec_slot, rec_capacity, dec_slot, dec_ballot, dec_shard_off, dec_data_len, dec_policy, dec_group,
                                   dec_capacity, pending, verdict, totals));
}
// Crossword soft fallback when a peer dies: unresponsive Accepting instances re-assigned `policy` and their codewords
// copied out for ss_frame_accept_pack_ragged_dev (see ss_engine_fallback_redo for the host contract and the cut)
inline void fallback_redo(ss_engine *e, const uint32_t *groups, uint64_t n_listed, const uint32_t *peer_alive, const uint8_t *policy,
                          uint8_t *shards, uint64_t plane_stride, uint64_t *store_used, uint64_t *dec_slot, uint64_t *dec_ballot,
                          uint64_t *dec_shard_off, uint32_t *dec_data_len, uint8_t *dec_policy, uint32_t *dec_group,
                          uint64_t dec_capacity, uint32_t *verdict, uint64_t *totals = nullptr) {
    check(ss_engine_fallback_redo(e, groups, n_listed, peer_alive, policy, shards, plane_stride, store_used, dec_slot, dec_ballot,
                                  dec_shard_off, dec_data_len, dec_policy, dec_group, dec_capacity, verdict, totals));
}
// step-down: the led bytes, and check_term over a batch of incoming frames (ss_engine_craft_step_down)
inline ss_engine_craft_role_view craft_role_view(ss_engine *e) {
    ss_engine_craft_role_view v{};
    check(ss_engine_craft_role_view_get(e, &v));
    return v;
}
inline void craft_step_down(ss_engine *e, Follower &follower, const ss_step_down_spec &spec, const uint8_t *buf, uint64_t buf_len,
                            const uint64_t *frame_off, const uint32_t *frame_group, const uint8_t *frame_peer, uint64_t n_frames,
                            uint8_t *store, uint64_t store_capacity, uint64_t *store_off, uint8_t *meta, uint32_t *meta_len,
                            uint32_t *verdict, uint64_t *need = nullptr) {
    check(ss_engine_craft_step_down(e, const_cast<ss_follower *>(follower.get()), &spec, buf, buf_len, frame_off, frame_group, frame_peer, n_frames, store,
                                    store_capacity, store_off, meta, meta_len, verdict, need));
}
inline void craft_reconstruct_reads(ss_engine *e, const uint32_t *groups, uint64_t n_listed, uint64_t chunk_size, uint8_t *out,
                                    uint64_t out_capacity, uint32_t *frame_group, uint8_t *frame_dst, uint64_t *frame_off,
                                    uint32_t *frame_len, uint64_t frame_capacity, uint64_t *totals = nullptr,
                                    uint32_t reconstruct_variant = 4) {
    check(ss_engine_craft_reconstruct_reads(e, groups, n_listed, chunk_size, reconstruct_variant, out, out_capacity, frame_group,
                                            frame_dst, frame_off, frame_len, frame_capacity, totals));
}
inline void craft_absorb(ss_engine *e, const uint8_t *buf, uint64_t buf_len, const uint64_t *frame_off, const uint32_t *frame_group,
                         const uint8_t *frame_peer, uint64_t n_frames, uint32_t *absorbed, uint32_t *verdict, uint32_t reply_variant = 5) {
    check(ss_engine_craft_absorb(e, buf, buf_len, frame_off, frame_group, frame_peer, n_frames, reply_variant, absorbed, verdict));
}

}  // namespace ssb
