"""ctypes binding of libsummerset_b200.so (the C ABI in include/summerset_b200.h).

Fails loudly when the shared library is missing: there is no Python / CPU fallback for any
compute entry point.  Build it with `python -m summerset_b200.build` (or __graft_entry__.build()).
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libsummerset_b200.so"

# error codes (include/summerset_b200.h)
SS_OK = 0
SS_ERR_TOO_FEW_SHARDS = -1
SS_ERR_TOO_MANY_SHARDS = -2
SS_ERR_TOO_FEW_DATA_SHARDS = -3
SS_ERR_TOO_MANY_DATA_SHARDS = -4
SS_ERR_TOO_FEW_PARITY_SHARDS = -5
SS_ERR_TOO_MANY_PARITY_SHARDS = -6
SS_ERR_INCORRECT_SHARD_SIZE = -9
SS_ERR_TOO_FEW_SHARDS_PRESENT = -10
SS_ERR_EMPTY_SHARD = -11
SS_ERR_INVALID_SHARD_FLAGS = -12
SS_ERR_INVALID_INDEX = -13
SS_ERR_INVALID_ARG = -20
SS_ERR_UNSUPPORTED = -21
SS_ERR_OUT_OF_MEMORY = -22
SS_ERR_NO_DEVICE = -30
SS_ERR_CUDA = -31
SS_RS_OUT_PADDED16 = 1

_vp, _u8p, _u32, _u64, _i = C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
_sz = C.c_size_t

# name -> (restype, argtypes); every symbol the header declares
SIGNATURES = {
    "ss_version": (_i, []),
    "ss_last_error": (C.c_char_p, []),
    "ss_strerror": (C.c_char_p, [_i]),
    "ss_ctx_create": (_i, [_i, C.POINTER(_vp)]),
    "ss_ctx_create_on_stream": (_i, [_i, _vp, C.POINTER(_vp)]),
    "ss_ctx_destroy": (_i, [_vp]),
    "ss_ctx_sync": (_i, [_vp]),
    "ss_ctx_stream": (_vp, [_vp]),
    "ss_ctx_sm_count": (_i, [_vp]),
    "ss_ctx_launch_count": (_u64, [_vp]),
    "ss_dev_alloc": (_i, [_vp, _sz, C.POINTER(_vp)]),
    "ss_dev_free": (_i, [_vp, _vp]),
    "ss_dev_memset": (_i, [_vp, _vp, _i, _sz]),
    "ss_host_alloc": (_i, [_vp, _sz, C.POINTER(_vp)]),
    "ss_host_alloc_wc": (_i, [_vp, _sz, C.POINTER(_vp)]),
    "ss_host_free": (_i, [_vp, _vp]),
    "ss_copy_h2d": (_i, [_vp, _vp, _vp, _sz]),
    "ss_copy_d2h": (_i, [_vp, _vp, _vp, _sz]),
    "ss_copy_d2d": (_i, [_vp, _vp, _vp, _sz]),
    "ss_ipc_export": (_i, [_vp, _vp, _vp]),
    "ss_ipc_open": (_i, [_vp, _vp, C.POINTER(_vp)]),
    "ss_ipc_close": (_i, [_vp, _vp]),
    "ss_accept_step_replicate_dev": (_i, [_vp, _vp, _u64, _u32, _u64, C.POINTER(_vp), _u64, _vp, _u32, _u32, _vp, _vp, _vp]),
    "ss_follower_ack_dev": (_i, [_vp, _vp, C.POINTER(_vp), _u32, _u64, _vp]),
    "ss_ctx_device_status": (_i, [_vp, C.POINTER(_u32)]),
    "ss_flags_wait_dev": (_i, [_vp, _vp]),
    "ss_flags_signal_dev": (_i, [_vp, _vp]),
    "ss_event_create": (_i, [_vp, C.POINTER(_vp)]),
    "ss_event_destroy": (_i, [_vp, _vp]),
    "ss_event_record": (_i, [_vp, _vp]),
    "ss_event_wait": (_i, [_vp, _vp]),
    "ss_rs_coder_create": (_i, [_vp, _i, _i, C.POINTER(_vp)]),
    "ss_rs_coder_destroy": (_i, [_vp]),
    "ss_rs_data_shard_count": (_i, [_vp]),
    "ss_rs_parity_shard_count": (_i, [_vp]),
    "ss_rs_total_shard_count": (_i, [_vp]),
    "ss_rs_coder_matrix": (_i, [_vp, _u8p]),
    "ss_rs_encode": (_i, [_vp, C.POINTER(_vp), _sz, _sz]),
    "ss_rs_reconstruct": (_i, [_vp, C.POINTER(_vp), _u8p, _sz, _sz]),
    "ss_rs_reconstruct_data": (_i, [_vp, C.POINTER(_vp), _u8p, _sz, _sz]),
    "ss_rs_verify": (_i, [_vp, C.POINTER(_vp), _sz, _sz, C.POINTER(_i)]),
    "ss_rs_encode_batch_dev": (_i, [_vp, _vp, _vp, _vp, _u64, _vp, _u64, _vp, _u32]),
    "ss_rs_encode_uniform_dev": (_i, [_vp, _vp, _u64, _u32, _u64, _vp, _u64, _u64, _u32]),
    "ss_rs_reconstruct_batch_dev": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _u64, _i, _vp, _u32]),
    "ss_rs_reconstruct_uniform_dev": (_i, [_vp, _vp, _u64, _u64, _u32, _vp, _u64, _i, _vp]),
    "ss_rs_encode_uniform": (_i, [_vp, _vp, _u64, _u32, _u64, _vp, _u64, _u64]),
    "ss_tally_planes_dev": (_i, [_vp, _vp, _u32, _u64, _u32, _vp, _vp]),
    "ss_tally_planes": (_i, [_vp, _vp, _u32, _u64, _u32, _vp, _vp]),
    "ss_tally_masks_dev": (_i, [_vp, _vp, _u32, _u64, _u32, _vp]),
    "ss_ack_ingest_dev": (_i, [_vp, _vp, _vp, _vp, _vp, _u64, _vp, _vp, _vp, _u32, _u64, _vp]),
    "ss_tally_crossword_dev": (_i, [_vp, _vp, _u32, _vp, _u64, _vp, _u32, _u32, _u32, _u32, _u32, _u32, _i, _vp]),
    "ss_raft_commit_scan_dev": (_i, [_vp, _vp, _u32, _u64, _vp, _vp, _vp, _vp, _u32, _u32, _vp, _vp]),
    "ss_crossword_distribute_dev": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _u64, C.POINTER(_vp), _u32]),
    "ss_frame_accept_batch_dev": (_i, [_vp, _vp, _u64, _u32, _u32, _u32, _u32, _u32, _vp, _vp, _u64, _vp, _u64, _vp, _vp]),
    "ss_gossip_plan_dev": (_i, [_vp, _u32, _u32, _u32, _vp, _vp, _vp, _vp, _u32, _u32, _u64, _vp, _vp]),
    "ss_raft_kth_match_dev": (_i, [_vp, _vp, _u32, _u64, _u32, _vp]),
    "ss_prepare_merge_dev": (_i, [_vp, _vp, _vp, _u32, _u64, _vp, _u32, _u32, _u32, _vp, _vp, _vp]),
    "ss_accept_step_fused_dev": (_i, [_vp, _vp, _u64, _u32, _u64, _vp, _u64, _u64, _u32, _vp, _u32, _u32, _vp, _vp]),
    "ss_accept_step_fused": (_i, [_vp, _vp, _u64, _u32, _u64, _vp, _u64, _u64, _vp, _u32, _u32, _vp, _vp]),
    "ss_frame_accept_max_len": (_u64, [_vp, _u32]),
    "ss_frame_accept_pack_dev": (_i, [_vp, _vp, _vp, _u64, _u64, _vp, _u32, _vp, _u32, _vp, _vp, _u64, _vp, _u64, _vp, _vp]),
    "ss_frame_accept_pack_ragged_dev": (_i, [_vp, _vp, _vp, _u64, _vp, _vp, _vp, _u32, _vp, _u32, _vp, _vp, _u64, _vp, _u64, _vp, _vp, _vp]),
    "ss_accept_reply_parse_dev": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _u64, _u32, _i, _vp, _vp, _vp, _vp, _vp]),
    "ss_wal_commit_pack_dev": (_i, [_vp, _vp, _vp, _u64, _u32, _vp, _vp, _vp, _u64, _vp]),
    "ss_reconstruct_serve_dev": (_i, [_vp, _vp, _u64, _u64, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _u64, _vp, _vp]),
    "ss_engine_create": (_i, [_vp, _vp, _u64, C.POINTER(_vp)]),
    "ss_engine_destroy": (_i, [_vp]),
    "ss_engine_view_get": (_i, [_vp, _vp]),
    "ss_engine_set_prepared_ballots": (_i, [_vp, _vp]),
    "ss_engine_set_policies": (_i, [_vp, _vp, _u32, _i]),
    "ss_engine_propose": (_i, [_vp, _u32, _vp, _u64, _vp, C.POINTER(_vp)]),
    "ss_engine_propose_next": (_i, [_vp, _u32, _vp, _u64, _vp, _vp, C.POINTER(_vp)]),
    "ss_engine_propose_ragged": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _u64, _vp, _vp, _vp]),
    "ss_engine_ingest": (_i, [_vp, _vp, _vp, _vp, _vp, _u64]),
    "ss_engine_tick": (_i, [_vp, _vp]),
    "ss_engine_advance": (_i, [_vp, _vp]),
    "ss_engine_window_get": (_i, [_vp, C.POINTER(_vp)]),
    "ss_engine_raft_append": (_i, [_vp, _vp]),
    "ss_engine_raft_ingest": (_i, [_vp, _vp, _vp, _vp, _u64]),
    "ss_acceptor_create": (_i, [_vp, _vp, _u64, C.POINTER(_vp)]),
    "ss_acceptor_destroy": (_i, [_vp]),
    "ss_acceptor_view_get": (_i, [_vp, _vp]),
    "ss_acceptor_window_get": (_i, [_vp, C.POINTER(_vp)]),
    "ss_acceptor_advance": (_i, [_vp, _vp]),
    "ss_acceptor_accept": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _u64, _vp, _u64, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ss_acceptor_commit_view_get": (_i, [_vp, _vp]),
    "ss_acceptor_heartbeat": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _u64, _vp]),
    "ss_acceptor_execute": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _vp]),
    "ss_acceptor_reconstruct_serve": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _u64, _u32, _u32, _vp, _u64, _vp, _vp, _vp, _vp]),
    "ss_acceptor_absorb": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _u64, _u32, _vp, _u64, _vp, _vp, _vp]),
    "ss_acceptor_prepare_view_get": (_i, [_vp, _vp]),
    "ss_acceptor_prepare": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _u64, _u32, _u32, _vp, _u64, _vp, _vp, _vp, _u64, _vp, _vp]),
    "ss_acceptor_prepare_reply": (_i, [_vp, _vp, _vp, _u64, _u32, _vp, _u64, _vp, _vp, _vp, _vp]),
    "ss_acceptor_recover": (_i, [_vp, _vp, _u64, _vp, _vp, _u64, _u32, _u32, _vp, _u64, _vp, _vp]),
    "ss_acceptor_gossip_view_get": (_i, [_vp, _vp]),
    "ss_acceptor_gossip": (_i, [_vp, _vp, _u64, _vp, _u64, _u64, _u32, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _vp]),
    "ss_acceptor_step_up_reads": (_i, [_vp, _vp, _u64, _u64, _u32, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _vp]),
    "ss_acceptor_step_up": (_i, [_vp, _vp, _u64, _u32, _u32, _vp, _u64, _vp, _vp, _u64, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _vp, _vp, _vp,
                                 _vp, _vp]),
    "ss_prepare_reply_parse_dev": (_i, [_vp, _vp, _u64, _vp, _u64, _u32, _u32, _u32, _vp]),
    "ss_engine_prepare_absorb": (_i, [_vp, _vp, _vp, _u64, _vp, _vp, _vp, _u64, _u32, _u32, _vp, _vp, _vp, _u64, _vp, _vp, _u64, _vp,
                                      _vp, _u64, _vp, _vp, _vp, _vp, _vp, _vp, _u64, _vp, _vp, _vp]),
    "ss_engine_fallback_redo": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _u64, _vp, _vp]),
    "ss_follower_create": (_i, [_vp, _vp, _u64, C.POINTER(_vp)]),
    "ss_follower_destroy": (_i, [_vp]),
    "ss_follower_view_get": (_i, [_vp, _vp]),
    "ss_follower_advance": (_i, [_vp, _vp]),
    "ss_follower_append": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _u64, _vp, _u64, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                _vp, _vp, _vp, _vp]),
    "ss_append_reply_parse_dev": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _u64, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ss_engine_craft_log_view_get": (_i, [_vp, _vp]),
    "ss_engine_craft_propose": (_i, [_vp, _u32, _vp, _vp, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _vp, _u64, _vp, _vp, _i]),
    "ss_engine_craft_advance": (_i, [_vp, _vp]),
    "ss_frame_append_pack_dev": (_i, [_vp, _vp, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _vp, _vp, _vp]),
    "ss_engine_craft_backoff": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _u32, _vp]),
    "ss_engine_craft_set_full_copy": (_i, [_vp, _i]),
    "ss_engine_craft_exec_view_get": (_i, [_vp, _vp]),
    "ss_engine_craft_execute": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _vp]),
    "ss_follower_exec_view_get": (_i, [_vp, _vp]),
    "ss_follower_execute": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _vp]),
    "ss_engine_craft_recon_view_get": (_i, [_vp, _vp]),
    "ss_engine_craft_step_up": (_i, [_vp, _vp, _vp, _u64, _vp, _vp, _u64, _vp, _vp, _vp]),
    "ss_engine_craft_reconstruct_reads": (_i, [_vp, _vp, _u64, _u64, _u32, _vp, _u64, _vp, _vp, _vp, _vp, _u64, _vp]),
    "ss_follower_reconstruct_serve": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _u64, _u32, _u32, _vp, _u64, _vp, _vp, _vp, _vp]),
    "ss_engine_craft_absorb": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _u64, _u32, _vp, _vp]),
    "ss_follower_vote_view_get": (_i, [_vp, _vp]),
    "ss_engine_craft_role_view_get": (_i, [_vp, _vp]),
    "ss_engine_craft_step_down": (_i, [_vp, _vp, _vp, _vp, _u64, _vp, _vp, _vp, _u64, _vp, _u64, _vp, _vp, _vp, _vp, _vp]),
    "ss_follower_campaign": (_i, [_vp, _vp, _u64, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ss_follower_vote": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _u64, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ss_follower_tally": (_i, [_vp, _vp, _u64, _vp, _vp, _vp, _u64, _u32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ss_follower_recover": (_i, [_vp, _vp, _u64, _vp, _vp, _u64, _vp, _u64, _vp, _vp]),
    "ss_rs_set_variant": (_i, [_vp, _i]),
    "ss_rs_last_kernel": (C.c_char_p, [_vp]),
    "ss_rs_jit_status": (C.c_char_p, [_vp]),
    "ss_jit_selftest": (C.c_long, [_i, _i, C.c_char_p, _sz]),
}


class StepSync(C.Structure):
    """ss_step_sync (include/summerset_b200.h): device-side wait / signal flags of one multi-GPU step call."""
    _fields_ = [("wait_flags", C.c_void_p), ("n_wait", C.c_uint32), ("wait_value", C.c_uint64),
                ("signal_flags", C.POINTER(C.c_void_p)), ("n_signal", C.c_uint32), ("signal_value", C.c_uint64)]


SS_PROTO_MULTIPAXOS, SS_PROTO_RSPAXOS, SS_PROTO_CROSSWORD, SS_PROTO_RAFT, SS_PROTO_CRAFT = range(5)


class FrameSpec(C.Structure):
    """ss_frame_spec"""
    _fields_ = [("kind", C.c_uint32), ("msg_variant", C.c_uint32), ("data_shards", C.c_uint32), ("parity_shards", C.c_uint32),
                ("data_len", C.c_uint32), ("population", C.c_uint32), ("with_assignment", C.c_uint32), ("assign_size", C.c_uint32)]


class EngineConfig(C.Structure):
    """ss_engine_config"""
    _fields_ = [("protocol", C.c_uint32), ("population", C.c_uint32), ("fault_tolerance", C.c_uint32), ("data_len", C.c_uint32),
                ("rs_total_shards", C.c_uint32), ("rs_data_shards", C.c_uint32), ("keep_slots", C.c_uint32),
                ("raft_window", C.c_uint32)]


class EngineView(C.Structure):
    """ss_engine_view"""
    _fields_ = [("n_groups", C.c_uint64), ("population", C.c_uint32), ("threshold", C.c_uint32), ("data_shards", C.c_uint32),
                ("total_shards", C.c_uint32), ("shard_len", C.c_uint32), ("shard_stride", C.c_uint32), ("raft_window", C.c_uint32),
                ("pad0", C.c_uint32), ("plane_stride", C.c_uint64), ("slot_stride", C.c_uint64),
                ("planes", C.c_void_p), ("bal_prepared", C.c_void_p), ("inst_bal", C.c_void_p), ("accepting", C.c_void_p),
                ("committed", C.c_void_p), ("commit_bar", C.c_void_p), ("shards", C.c_void_p), ("policy_idx", C.c_void_p),
                ("match", C.c_void_p), ("next_slot", C.c_void_p), ("last_commit", C.c_void_p), ("log_end", C.c_void_p),
                ("curr_term", C.c_void_p), ("last_snap", C.c_void_p), ("terms", C.c_void_p)]


class AcceptorConfig(C.Structure):
    """ss_acceptor_config"""
    _fields_ = [("protocol", C.c_uint32), ("population", C.c_uint32), ("me", C.c_uint32), ("data_shards", C.c_uint32),
                ("total_shards", C.c_uint32), ("accept_variant", C.c_uint32), ("wal_variant", C.c_uint32), ("reply_variant", C.c_uint32)]


class AcceptorView(C.Structure):
    """ss_acceptor_view"""
    _fields_ = [("n_groups", C.c_uint64), ("protocol", C.c_uint32), ("population", C.c_uint32), ("me", C.c_uint32),
                ("data_shards", C.c_uint32), ("total_shards", C.c_uint32), ("pad0", C.c_uint32),
                ("window_base", C.c_void_p), ("bal_max_seen", C.c_void_p), ("inst_bal", C.c_void_p), ("accepting", C.c_void_p),
                ("shard_addr", C.c_void_p), ("held", C.c_void_p), ("data_len", C.c_void_p), ("assignment", C.c_void_p),
                ("source", C.c_void_p)]


class AcceptorCommitView(C.Structure):
    """ss_acceptor_commit_view"""
    _fields_ = [("n_groups", C.c_uint64), ("committed", C.c_void_p), ("commit_bar", C.c_void_p), ("exec_bar", C.c_void_p)]


class AcceptorPrepareView(C.Structure):
    """ss_acceptor_prepare_view"""
    _fields_ = [("n_groups", C.c_uint64), ("preparing", C.c_void_p), ("voted_bal", C.c_void_p), ("voted_mask", C.c_void_p),
                ("prep_trigger", C.c_void_p), ("prep_span", C.c_void_p)]


class AcceptorGossipView(C.Structure):
    """ss_acceptor_gossip_view"""
    _fields_ = [("n_groups", C.c_uint64), ("population", C.c_uint32), ("pad0", C.c_uint32), ("assign_rows", C.c_void_p),
                ("gossip_bar", C.c_void_p)]


class FollowerConfig(C.Structure):
    """ss_follower_config"""
    _fields_ = [("protocol", C.c_uint32), ("population", C.c_uint32), ("me", C.c_uint32), ("window", C.c_uint32),
                ("append_variant", C.c_uint32), ("reply_variant", C.c_uint32), ("meta_variant", C.c_uint32),
                ("log_variant", C.c_uint32)]


class FollowerView(C.Structure):
    """ss_follower_view"""
    _fields_ = [("n_groups", C.c_uint64), ("protocol", C.c_uint32), ("population", C.c_uint32), ("me", C.c_uint32),
                ("data_shards", C.c_uint32), ("total_shards", C.c_uint32), ("window", C.c_uint32),
                ("start_slot", C.c_void_p), ("log_end", C.c_void_p), ("curr_term", C.c_void_p), ("last_commit", C.c_void_p),
                ("last_snap", C.c_void_p), ("leader", C.c_void_p), ("term", C.c_void_p), ("shard_addr", C.c_void_p),
                ("held", C.c_void_p), ("data_len", C.c_void_p)]


class CraftLogView(C.Structure):
    """ss_engine_craft_log_view"""
    _fields_ = [("n_groups", C.c_uint64), ("population", C.c_uint32), ("raft_window", C.c_uint32), ("data_shards", C.c_uint32),
                ("total_shards", C.c_uint32), ("plane_stride", C.c_uint64), ("log_start", C.c_void_p), ("try_next", C.c_void_p),
                ("data_len", C.c_void_p), ("shard_addr", C.c_void_p), ("log_offset", C.c_void_p)]


class CraftExecView(C.Structure):
    """ss_engine_craft_exec_view"""
    _fields_ = [("n_groups", C.c_uint64), ("last_exec", C.c_void_p)]


class CraftReconView(C.Structure):
    """ss_engine_craft_recon_view"""
    _fields_ = [("n_groups", C.c_uint64), ("raft_window", C.c_uint32), ("total_shards", C.c_uint32), ("held", C.c_void_p),
                ("last_recon", C.c_void_p)]


class CraftRoleView(C.Structure):
    """ss_engine_craft_role_view"""
    _fields_ = [("n_groups", C.c_uint64), ("led", C.c_void_p)]


class StepDownSpec(C.Structure):
    """ss_step_down_spec"""
    _fields_ = [("append_variant", C.c_uint32), ("append_reply_variant", C.c_uint32), ("request_vote_variant", C.c_uint32),
                ("vote_reply_variant", C.c_uint32)]


class FollowerExecView(C.Structure):
    """ss_follower_exec_view"""
    _fields_ = [("n_groups", C.c_uint64), ("last_exec", C.c_void_p)]


class FollowerVoteView(C.Structure):
    """ss_follower_vote_view"""
    _fields_ = [("n_groups", C.c_uint64), ("vote_term", C.c_void_p), ("voted_for", C.c_void_p), ("role_term", C.c_void_p),
                ("role", C.c_void_p), ("votes", C.c_void_p)]


class AppendPackSpec(C.Structure):
    """ss_append_pack_spec"""
    _fields_ = [("me", C.c_uint32), ("append_variant", C.c_uint32), ("msg_chunk_size", C.c_uint32), ("full_copy", C.c_uint32),
                ("heartbeat", C.c_uint32), ("pad0", C.c_uint32)]


class PrepareReplyRec(C.Structure):
    """ss_prepare_reply_rec (64 bytes)"""
    _fields_ = [("slot", C.c_uint64), ("trigger_slot", C.c_uint64), ("endprep_slot", C.c_uint64), ("ballot", C.c_uint64),
                ("vote_bal", C.c_uint64), ("shards_at", C.c_uint64), ("vote_mask", C.c_uint32), ("data_len", C.c_uint32),
                ("kind", C.c_uint32), ("pad", C.c_uint32)]


# the execution walks' bits of the device status word (ss_acceptor_execute, ss_follower_execute, ss_engine_craft_execute)
SS_DEV_STATUS_EXEC_FULL = 32
SS_DEV_STATUS_EXEC_NULL = 64

# verdicts of ss_acceptor_accept (beside PeerMsg variant indices and SS_FRAME_KIND_MALFORMED)
SS_ACCEPT_VERDICT_ACCEPTED = 0xFFFFFFF0
SS_ACCEPT_VERDICT_STALE_SLOT = 0xFFFFFFF1
SS_ACCEPT_VERDICT_STALE_BALLOT = 0xFFFFFFF2
SS_ACCEPT_VERDICT_BEYOND_WINDOW = 0xFFFFFFF3
SS_ACCEPT_VERDICT_STORE_FULL = 0xFFFFFFF4
SS_ACCEPT_VERDICT_WAL_FULL = 0xFFFFFFF5
SS_FRAME_KIND_MALFORMED = 0xFFFFFFFF
# verdicts of ss_acceptor_reconstruct_serve beside those above
SS_RECON_VERDICT_NULL_CODEWORD = 0xFFFFFFF6
SS_RECON_VERDICT_SHARD_RANGE = 0xFFFFFFF7
SS_RECON_VERDICT_OUT_FULL = 0xFFFFFFF8
# verdict of ss_acceptor_recover beside the accept verdicts: after a malformed record of its group
SS_RECOVER_VERDICT_AFTER_END = 0xFFFFFFF9
# verdicts of ss_follower_append (beside PeerMsg variant indices and SS_FRAME_KIND_MALFORMED)
SS_FOLLOWER_VERDICT_ACCEPTED = 0xFFFFFFF0
SS_FOLLOWER_VERDICT_REJECTED = 0xFFFFFFF1
SS_FOLLOWER_VERDICT_BEYOND_WINDOW = 0xFFFFFFF3
SS_FOLLOWER_VERDICT_STORE_FULL = 0xFFFFFFF4
SS_FOLLOWER_VERDICT_WAL_FULL = 0xFFFFFFF5
# record kinds of ss_append_reply_parse_dev
SS_APPEND_REPLY_INGEST = 0xFFFFFFF0
SS_APPEND_REPLY_CONFLICT = 0xFFFFFFF1
SS_APPEND_REPLY_HIGHER_TERM = 0xFFFFFFF2
SS_APPEND_REPLY_END_RANGE = 0xFFFFFFF3
# verdicts of ss_engine_prepare_absorb, beside the acceptor's
SS_PREP_VERDICT_IGNORED = 0xFFFFFFFA
SS_PREP_VERDICT_DATA_LEN = 0xFFFFFFFB
# verdicts of ss_engine_craft_step_up
SS_STEPUP_VERDICT_DONE, SS_STEPUP_VERDICT_IGNORED, SS_STEPUP_VERDICT_WINDOW, SS_STEPUP_VERDICT_RANGE, \
    SS_STEPUP_VERDICT_STALE_TERM, SS_STEPUP_VERDICT_STORE_FULL = range(6)
# CRaft elections: follower roles, verdicts of ss_follower_campaign, ss_follower_vote and ss_follower_tally
SS_FOLLOWER_ROLE_FOLLOWER, SS_FOLLOWER_ROLE_CANDIDATE, SS_FOLLOWER_ROLE_ELECTED = range(3)
SS_CAMPAIGN_VERDICT_DONE, SS_CAMPAIGN_VERDICT_IGNORED, SS_CAMPAIGN_VERDICT_NOT_FOLLOWER, SS_CAMPAIGN_VERDICT_OTHER_LEADER, \
    SS_CAMPAIGN_VERDICT_RANGE = range(5)
SS_VOTE_VERDICT_GRANTED, SS_VOTE_VERDICT_DENIED_STALE, SS_VOTE_VERDICT_NO_REPLY = range(0xFFFFFFF0, 0xFFFFFFF3)
SS_TALLY_VERDICT_HIGHER_TERM, SS_TALLY_VERDICT_ELECTED_ALREADY, SS_TALLY_VERDICT_NOT_CANDIDATE, SS_TALLY_VERDICT_STALE_TERM, \
    SS_TALLY_VERDICT_DENIED, SS_TALLY_VERDICT_DUPLICATE, SS_TALLY_VERDICT_COUNTED, SS_TALLY_VERDICT_WON = range(0xFFFFFFF0, 0xFFFFFFF8)
# pair statuses of ss_frame_append_pack_dev
SS_APPEND_PAIR_SENT, SS_APPEND_PAIR_NOTHING, SS_APPEND_PAIR_SNAPSHOTTED, SS_APPEND_PAIR_OVERFLOW, SS_APPEND_PAIR_NOT_LEADER = range(5)
# CRaft step-down: verdicts of ss_engine_craft_step_down, and the status bit of a call refused for a group not led
SS_STEPDOWN_VERDICT_PASS, SS_STEPDOWN_VERDICT_RANGE, SS_STEPDOWN_VERDICT_STORE_FULL, SS_STEPDOWN_VERDICT_DEPOSED = range(0xFFFFFFF0, 0xFFFFFFF4)
SS_DEV_STATUS_NOT_LEADER = 128


class SummersetError(RuntimeError):
    """Mirror of `SummersetError(String)` (src/utils/error.rs:6-14): message + the C error code."""

    def __init__(self, code: int, msg: str):
        super().__init__(f"[{code}] {msg}")
        self.code = code
        self.msg = msg


_lib = None


def load() -> C.CDLL:
    """Loads the shared library and binds every declared symbol. Raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise ImportError(
            f"{LIB_PATH} is missing: build the CUDA extension first "
            "(`python -m summerset_b200.build`); there is no CPU fallback")
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != SS_OK:
        lib = load()
        msg = lib.ss_last_error().decode("utf-8", "replace")
        raise SummersetError(rc, msg or lib.ss_strerror(rc).decode())
