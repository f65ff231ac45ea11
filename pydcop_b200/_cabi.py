"""ctypes binding of include/pydcop_b200.h (the C-ABI of libpydcop_b200.so).

Fails loudly when the library is missing: there is no Python/CPU fallback for the hot path.
"""
import ctypes as C
import os

FG_ABI_VERSION = 3
FG_MAX_ARITY = 8
FG_MAX_DOM = 256
FG_OK, FG_ERR_ARG, FG_ERR_CUDA, FG_ERR_UNSUPPORTED = 0, 1, 2, 3
FG_F32, FG_F64 = 0, 1
START_MESSAGES = {"leafs": 0, "leafs_vars": 1, "all": 2}
DSA_VARIANTS = {"A": 0, "B": 1, "C": 2}
FG_MAX_PSETS = 65535   # parameter sets of one handle (uint16 indices)

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libpydcop_b200.so")


class FgClass(C.Structure):
    _fields_ = [("arity", C.c_int32), ("dom", C.c_int32 * FG_MAX_ARITY),
                ("row_off", C.c_int32 * FG_MAX_ARITY), ("row_total", C.c_int32),
                ("n_factors", C.c_int32), ("flags", C.c_int32), ("first_factor", C.c_int32),
                ("first_edge", C.c_int32),
                ("table_size", C.c_int64), ("table_base", C.c_int64), ("msg_base", C.c_int64)]


P = C.c_void_p


class FgVarClass(C.Structure):
    _fields_ = [("dom", C.c_int32), ("degree", C.c_int32), ("n_vars", C.c_int32),
                ("first_var", C.c_int32), ("first_slot", C.c_int32), ("n_slots", C.c_int32),
                ("flags", C.c_int32), ("reserved", C.c_int32),
                ("unary_base", C.c_int64), ("q_base", C.c_int64)]


class FgMaxSumDesc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("precision", C.c_int32),
                ("n_vars", C.c_int32), ("n_factors", C.c_int32), ("n_edges", C.c_int32),
                ("n_classes", C.c_int32), ("n_msg_r", C.c_int64), ("n_msg_q", C.c_int64),
                ("uniform_dom", C.c_int32), ("max_degree", C.c_int32),
                ("classes", C.POINTER(FgClass)),
                ("n_varclasses", C.c_int32), ("reserved0", C.c_int32),
                ("varclasses", C.POINTER(FgVarClass)),
                ("dev_tables", P), ("dev_unary", P), ("dev_dom_size", P), ("dev_unary_off", P),
                ("dev_var_ptr", P), ("dev_var_qbase", P), ("dev_slot_roff", P), ("dev_edge_qoff", P),
                ("dev_slot_roff32", P), ("dev_edge_qoff32", P),
                ("dev_slot_edge", P), ("dev_slot_var", P),
                ("dev_init_value", P),
                ("dev_q", P * 2), ("dev_r", P * 2), ("dev_q_valid", P), ("dev_r_valid", P),
                ("dev_q_cnt", P), ("dev_r_cnt", P), ("dev_q_sent", P), ("dev_r_sent", P),
                ("dev_value", P), ("dev_value_cost", P),
                ("mode_max", C.c_int32), ("damp_vars", C.c_int32), ("damp_factors", C.c_int32),
                ("start_messages", C.c_int32), ("damping", C.c_double), ("stability", C.c_double)]


class FgDsaPset(C.Structure):
    _fields_ = [("variant", C.c_int32)]


class FgDsaDesc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("precision", C.c_int32),
                ("n_vars", C.c_int32), ("n_factors", C.c_int32), ("n_edges", C.c_int32),
                ("n_classes", C.c_int32), ("classes", C.POINTER(FgClass)),
                ("dev_tables", P), ("dev_dom_size", P), ("dev_var_id", P), ("dev_edge_var", P),
                ("dev_edge_class", P),
                ("dev_var_ptr", P), ("dev_slot_edge", P), ("dev_has_nbr", P), ("dev_prob", P),
                ("dev_con_opt", P), ("dev_tables_or", P), ("dev_slot_nbr", P), ("dev_slot_tab", P),
                ("dev_slot_opt", P), ("fast_dom", C.c_int32), ("reserved1", C.c_int32),
                ("dev_value", P * 2), ("dev_value_cost", P),
                ("mode_max", C.c_int32), ("variant", C.c_int32), ("stop_cycle", C.c_int32),
                ("seed", C.c_uint64), ("dev_var_cost", P), ("dev_unary_off", P),
                ("dev_row_cache", P), ("dev_slot_last", P),
                ("dev_var_seed", P),
                ("dev_var_pset", P), ("psets", C.POINTER(FgDsaPset)), ("n_psets", C.c_int32),
                ("reserved_ps", C.c_int32)]


class FgMgmDesc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("precision", C.c_int32),
                ("n_vars", C.c_int32), ("n_factors", C.c_int32), ("n_edges", C.c_int32),
                ("n_classes", C.c_int32), ("classes", C.POINTER(FgClass)),
                ("dev_tables", P), ("dev_unary", P), ("dev_unary_off", P), ("dev_dom_size", P),
                ("dev_var_id", P), ("dev_var_rank", P), ("dev_edge_var", P), ("dev_edge_class", P),
                ("dev_var_ptr", P), ("dev_slot_edge", P), ("dev_nbr_ptr", P), ("dev_nbr_idx", P),
                ("dev_init_value", P), ("dev_value", P), ("dev_cost", P), ("dev_has_cost", P),
                ("dev_gain", P), ("dev_new_value", P),
                ("mode_max", C.c_int32), ("stop_cycle", C.c_int32), ("seed", C.c_uint64),
                ("dev_tables_or", P), ("dev_slot_nbr", P), ("dev_slot_tab", P),
                ("fast_dom", C.c_int32), ("fast_chunk", C.c_int32),
                ("dev_row_cache", P), ("dev_slot_last", P),
                ("dev_var_seed", P)]


class FgMgm2Pset(C.Structure):
    _fields_ = [("threshold", C.c_double), ("favor", C.c_int32), ("reserved0", C.c_int32)]


class FgMgm2Desc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("precision", C.c_int32),
                ("n_vars", C.c_int32), ("n_factors", C.c_int32), ("n_edges", C.c_int32),
                ("n_classes", C.c_int32), ("classes", C.POINTER(FgClass)),
                ("dev_tables", P), ("dev_dom_size", P), ("dev_var_id", P), ("dev_var_rank", P),
                ("dev_edge_var", P), ("dev_edge_class", P), ("dev_var_ptr", P), ("dev_slot_edge", P),
                ("dev_nbr_ptr", P), ("dev_nbr_idx", P), ("dev_init_value", P),
                ("dev_value", P), ("dev_cost", P), ("dev_has_cost", P), ("dev_gain", P),
                ("dev_potential_value", P), ("dev_local_cost", P), ("dev_offerer", P), ("dev_partner", P),
                ("dev_committed", P), ("dev_go", P), ("dev_answer", P), ("dev_answer_value", P),
                ("dev_answer_gain", P), ("dev_offer_off", P), ("dev_offer", P),
                ("mode_max", C.c_int32), ("favor", C.c_int32), ("threshold", C.c_double),
                ("stop_cycle", C.c_int32), ("reserved0", C.c_int32), ("seed", C.c_uint64),
                ("dev_var_seed", P),
                ("dev_var_pset", P), ("psets", C.POINTER(FgMgm2Pset)), ("n_psets", C.c_int32),
                ("reserved_ps", C.c_int32)]


MGM2_FAVORS = {"unilateral": 0, "no": 1, "coordinated": 2}


class FgGdbaPset(C.Structure):
    _fields_ = [("modifier", C.c_int32), ("violation", C.c_int32)]


class FgGdbaDesc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("precision", C.c_int32),
                ("n_vars", C.c_int32), ("n_factors", C.c_int32), ("n_edges", C.c_int32),
                ("n_classes", C.c_int32), ("classes", C.POINTER(FgClass)),
                ("dev_tables", P), ("dev_unary", P), ("dev_unary_off", P), ("dev_viol_ref", P),
                ("dev_dom_size", P), ("dev_var_id", P), ("dev_var_rank", P),
                ("dev_edge_var", P), ("dev_edge_class", P), ("dev_var_ptr", P), ("dev_slot_edge", P),
                ("dev_nbr_ptr", P), ("dev_nbr_idx", P), ("dev_init_value", P),
                ("dev_value", P * 2), ("dev_cost", P), ("dev_has_cost", P), ("dev_improve", P),
                ("dev_new_value", P), ("dev_violated", P), ("dev_breakout", P), ("dev_mod", P), ("dev_mod_off", P),
                ("mode_max", C.c_int32), ("modifier", C.c_int32), ("violation", C.c_int32),
                ("increase_mode", C.c_int32), ("stop_cycle", C.c_int32), ("reserved0", C.c_int32),
                ("mod_size", C.c_int64), ("seed", C.c_uint64),
                ("dev_var_seed", P),
                ("dev_var_pset", P), ("psets", C.POINTER(FgGdbaPset)), ("n_psets", C.c_int32),
                ("reserved_ps", C.c_int32)]


class FgDpopLaunch(C.Structure):
    _fields_ = [("kind", C.c_int32), ("first", C.c_int32), ("count", C.c_int32), ("reserved", C.c_int32)]


class FgDpopDesc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("precision", C.c_int32),
                ("n_vars", C.c_int32), ("mode_max", C.c_int32),
                ("n_terms", C.c_int64), ("n_tdims", C.c_int64), ("arena_size", C.c_int64),
                ("dev_unary", P), ("dev_tables", P), ("dev_arena", P),
                ("dev_dom_size", P), ("dev_unary_off", P), ("dev_util_off", P), ("dev_util_size", P),
                ("dev_sep_ptr", P), ("dev_sep_var", P), ("dev_term_ptr", P), ("dev_term_kind", P),
                ("dev_term_base", P), ("dev_term_own", P), ("dev_tdim_ptr", P), ("dev_tdim_pos", P),
                ("dev_tdim_stride", P), ("dev_util_nodes", P), ("dev_util_seg_ptr", P),
                ("dev_value_nodes", P), ("dev_value_seg_ptr", P),
                ("n_util_segs", C.c_int32), ("n_value_segs", C.c_int32),
                ("n_util_launches", C.c_int32), ("n_value_launches", C.c_int32),
                ("util_launches", C.POINTER(FgDpopLaunch)), ("value_launches", C.POINTER(FgDpopLaunch)),
                ("dev_value", P), ("dev_cost", P), ("dev_unresolved", P),
                ("max_sep", C.c_int32), ("reserved0", C.c_int32)]


class FgDbaDesc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("precision", C.c_int32),
                ("n_vars", C.c_int32), ("n_factors", C.c_int32), ("n_edges", C.c_int32),
                ("n_classes", C.c_int32), ("classes", C.POINTER(FgClass)),
                ("dev_tables", P), ("dev_dom_size", P), ("dev_var_id", P), ("dev_var_rank", P),
                ("dev_edge_var", P), ("dev_edge_class", P), ("dev_var_ptr", P), ("dev_slot_edge", P),
                ("dev_nbr_ptr", P), ("dev_nbr_idx", P), ("dev_bit_off", P), ("dev_bits", P),
                ("dev_value", P * 2), ("dev_cost", P), ("dev_has_cost", P), ("dev_eval", P), ("dev_improve", P),
                ("dev_counter", P), ("dev_counter_own", P), ("dev_new_value", P),
                ("dev_can_move", P), ("dev_qlm", P), ("dev_consistent", P), ("dev_finish_phase", P),
                ("dev_weight", P), ("dev_violated", P), ("dev_status", P), ("dev_unresolved", P),
                ("n_words", C.c_int64), ("infinity", C.c_int64),
                ("max_distance", C.c_int32), ("stop_cycle", C.c_int32), ("n_live", C.c_int32),
                ("reserved0", C.c_int32), ("seed", C.c_uint64)]


class FgSyncbbDesc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("precision", C.c_int32), ("n_vars", C.c_int32), ("mode_max", C.c_int32),
                ("dev_dom", P), ("dev_elt_ptr", P), ("dev_elt_pos", P), ("dev_elt_tab", P), ("dev_pair", P),
                ("dev_ub", P), ("dev_sel", P), ("dev_path_val", P), ("dev_path_cost", P), ("dev_path_sum", P),
                ("dev_path_comp", P), ("dev_msg", P), ("dev_msg_ub", P), ("dev_count", P),
                ("dev_cycles", P), ("n_elts", C.c_int64), ("n_pair", C.c_int64)]


class FgMixedDsaPset(C.Structure):
    _fields_ = [("proba_hard", C.c_double), ("proba_soft", C.c_double), ("variant", C.c_int32),
                ("reserved0", C.c_int32)]


class FgMixedDsaDesc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("precision", C.c_int32),
                ("n_vars", C.c_int32), ("n_factors", C.c_int32), ("n_edges", C.c_int32),
                ("n_classes", C.c_int32), ("classes", C.POINTER(FgClass)),
                ("dev_tables", P), ("dev_unary", P), ("dev_unary_off", P), ("dev_dom_size", P), ("dev_var_id", P),
                ("dev_edge_var", P), ("dev_edge_class", P), ("dev_var_ptr", P), ("dev_slot_edge", P),
                ("dev_soft_end", P), ("dev_nbr_ptr", P), ("dev_nbr_idx", P), ("dev_init_value", P),
                ("dev_con_opt", P), ("dev_value", P * 2), ("dev_cost", P), ("dev_has_cost", P),
                ("dev_h_best", P), ("dev_branch", P),
                ("proba_hard", C.c_double), ("proba_soft", C.c_double),
                ("mode_max", C.c_int32), ("variant", C.c_int32), ("stop_cycle", C.c_int32),
                ("reserved0", C.c_int32), ("seed", C.c_uint64), ("dev_var_seed", P),
                ("dev_var_pset", P), ("psets", C.POINTER(FgMixedDsaPset)), ("n_psets", C.c_int32),
                ("reserved_ps", C.c_int32)]


MIXEDDSA_VARIANTS = {"A": 0, "B": 1, "C": 2}
# fg_mixeddsa_desc_t dev_branch: the case of mixeddsa.py:300-358 that applied, | MIXEDDSA_MOVED
MIXEDDSA_BRANCH_NONE, MIXEDDSA_BRANCH_HARD, MIXEDDSA_BRANCH_SOFT = 0, 1, 2
MIXEDDSA_BRANCH_STUCK_HARD, MIXEDDSA_BRANCH_STUCK_SOFT, MIXEDDSA_BRANCH_IDLE = 3, 4, 5
MIXEDDSA_MOVED = 8

GDBA_MODIFIERS = {"A": 0, "M": 1}
GDBA_VIOLATIONS = {"NZ": 0, "NM": 1, "MX": 2}
GDBA_INCREASE_MODES = {"E": 0, "R": 1, "C": 2, "T": 3}

FG_MAX_PEERS = 16


class FgPeerSync(C.Structure):
    _fields_ = [("n_peers", C.c_int32), ("my_rank", C.c_int32), ("dev_flags", P),
                ("peer_rank", C.c_int32 * FG_MAX_PEERS), ("peer_slot", P * FG_MAX_PEERS),
                ("dev_error", P), ("timeout_ns", C.c_uint64)]


class FgHaloPlan(C.Structure):
    _fields_ = [("elem_bytes", C.c_int32), ("dom", C.c_int32), ("n_r", C.c_int64), ("n_q", C.c_int64),
                ("dev_src_r_off", P), ("dev_src_q_off", P), ("dev_dst_r", P * 2), ("dev_dst_q", P * 2),
                ("dev_counter", P), ("sync", FgPeerSync),
                ("dev_runs_r", P * 2), ("dev_runs_q", P * 2), ("n_runs_r", C.c_int32 * 2), ("n_runs_q", C.c_int32 * 2),
                ("units_r", C.c_int64 * 2), ("units_q", C.c_int64 * 2),
                ("dev_edge_dst_r", P * 2), ("dev_slot_dst_q", P * 2)]


class FgTraceDesc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("precision", C.c_int32), ("n_vars", C.c_int32), ("n_classes", C.c_int32),
                ("classes", C.POINTER(FgClass)), ("dev_tables", P), ("dev_edge_var", P), ("dev_unary", P),
                ("dev_unary_off", P), ("dev_factor_seg", P), ("dev_var_seg", P),
                ("n_seg", C.c_int32), ("reserved0", C.c_int32), ("infinity", C.c_double),
                ("dev_rows", P), ("dev_stamp", P), ("capacity", C.c_int64)]


FG_MGM2_EXCHANGES = 5


class FgMgm2Xfer(C.Structure):
    _fields_ = [("n_send", C.c_int64), ("n_recv", C.c_int64), ("dev_send_var", P), ("dev_recv_var", P),
                ("dev_send_off", P), ("dev_recv_off", P), ("dev_send_buf", P), ("dev_recv_buf", P)]


class FgMgm2ShardPlan(C.Structure):
    _fields_ = [("x", FgMgm2Xfer * FG_MGM2_EXCHANGES), ("dev_ghost", P), ("dev_send_peer", P),
                ("dev_owner_rank", P), ("dev_owner_local", P)]


class FgMgm2PeerPlan(C.Structure):
    _fields_ = [("n_blocks", C.c_int32 * FG_MGM2_EXCHANGES), ("reserved0", C.c_int32),
                ("src", (C.c_int64 * FG_MAX_PEERS) * FG_MGM2_EXCHANGES),
                ("n_elems", (C.c_int64 * FG_MAX_PEERS) * FG_MGM2_EXCHANGES),
                ("dst", (C.c_uint64 * FG_MAX_PEERS) * FG_MGM2_EXCHANGES),
                ("dev_counter", P), ("sync", FgPeerSync)]

# every symbol include/pydcop_b200.h declares: (restype, argtypes)
SYMBOLS = {
    "fg_abi_version": (C.c_int, []),
    "fg_device_count": (C.c_int, []),
    "fg_maxsum_create": (C.c_int, [C.POINTER(FgMaxSumDesc), C.POINTER(P)]),
    "fg_maxsum_destroy": (C.c_int, [P]),
    "fg_maxsum_last_error": (C.c_char_p, [P]),
    "fg_maxsum_init": (C.c_int, [P, P]),
    "fg_maxsum_step": (C.c_int, [P, C.c_int32, P]),
    "fg_maxsum_cycle_compute": (C.c_int, [P, P]),
    "fg_maxsum_cycle_commit": (C.c_int, [P]),
    "fg_maxsum_current": (C.c_int, [P, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "fg_maxsum_launch_count": (C.c_int64, [P]),
    "fg_maxsum_kernel_plan": (C.c_int, [P, P, C.c_int32]),
    "fg_maxsum_table_width": (C.c_int, [P, P, C.c_int32]),
    "fg_maxsum_shard_fused": (C.c_int, [P]),
    "fg_halo_pack": (C.c_int, [C.c_int32, P, P, P, P, P, C.c_int64, P]),
    "fg_halo_unpack": (C.c_int, [C.c_int32, P, P, P, P, P, C.c_int64, P]),
    "fg_halo_rows_uniform": (C.c_int, [C.c_int32, C.c_int32, P, P, P, P, P, C.c_int64, C.c_int64,
                                       C.c_int32, C.c_int32, P, P, P, P]),
    "fg_enable_peer_access": (C.c_int, [C.c_int32]),
    "fg_ipc_export": (C.c_int, [P, P, C.POINTER(C.c_int64)]),
    "fg_ipc_import": (C.c_int, [P, C.POINTER(P)]),
    "fg_ipc_close": (C.c_int, [P]),
    "fg_halo_push": (C.c_int, [C.c_int32, P, P, P, P, P, P, C.c_int64, C.c_int64, C.c_int32, P]),
    "fg_peer_signal": (C.c_int, [C.POINTER(FgPeerSync), C.c_uint64, P]),
    "fg_peer_wait": (C.c_int, [C.POINTER(FgPeerSync), C.c_uint64, P]),
    "fg_maxsum_shard_attach": (C.c_int, [P, C.POINTER(FgHaloPlan)]),
    "fg_maxsum_shard_step": (C.c_int, [P, C.c_int32, P]),
    "fg_maxsum_shard_phase": (C.c_int, [P, C.c_int32, P]),
    "fg_maxsum_shard_profile": (C.c_int, [P, C.c_int32, P, C.POINTER(C.c_double)]),
    "fg_dsa_shard_attach": (C.c_int, [P, C.POINTER(FgHaloPlan)]),
    "fg_dsa_shard_step": (C.c_int, [P, C.c_int32, P]),
    "fg_dsa_create": (C.c_int, [C.POINTER(FgDsaDesc), C.POINTER(P)]),
    "fg_dsa_destroy": (C.c_int, [P]),
    "fg_dsa_last_error": (C.c_char_p, [P]),
    "fg_dsa_init": (C.c_int, [P, P]),
    "fg_dsa_step": (C.c_int, [P, C.c_int32, P]),
    "fg_dsa_cycle_compute": (C.c_int, [P, P]),
    "fg_dsa_cycle_commit": (C.c_int, [P]),
    "fg_dsa_current": (C.c_int, [P, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "fg_dsa_launch_count": (C.c_int64, [P]),
    "fg_selftest_approx_match": (C.c_int, [C.c_int32, C.c_int64, P, P, C.c_double, P, P, P]),
    "fg_selftest_gather": (C.c_int, [P, C.c_int64, C.c_int32, C.c_int32, C.c_int64, C.c_int32, P, P]),
    "fg_mgm_create": (C.c_int, [C.POINTER(FgMgmDesc), C.POINTER(P)]),
    "fg_mgm_destroy": (C.c_int, [P]),
    "fg_mgm_last_error": (C.c_char_p, [P]),
    "fg_mgm_init": (C.c_int, [P, P]),
    "fg_mgm_step": (C.c_int, [P, C.c_int32, P]),
    "fg_mgm_current": (C.c_int, [P, C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "fg_mgm_launch_count": (C.c_int64, [P]),
    "fg_mgm2_create": (C.c_int, [C.POINTER(FgMgm2Desc), C.POINTER(P)]),
    "fg_mgm2_destroy": (C.c_int, [P]),
    "fg_mgm2_last_error": (C.c_char_p, [P]),
    "fg_mgm2_init": (C.c_int, [P, P]),
    "fg_mgm2_step": (C.c_int, [P, C.c_int32, P]),
    "fg_mgm2_current": (C.c_int, [P, C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "fg_mgm2_launch_count": (C.c_int64, [P]),
    "fg_mgm2_shard_attach": (C.c_int, [P, C.POINTER(FgMgm2ShardPlan), C.POINTER(FgMgm2PeerPlan)]),
    "fg_mgm2_shard_init": (C.c_int, [P, P]),
    "fg_mgm2_shard_phase": (C.c_int, [P, C.c_int32, P]),
    "fg_mgm2_shard_unpack": (C.c_int, [P, C.c_int32, P]),
    "fg_mgm2_shard_step": (C.c_int, [P, C.c_int32, P]),
    "fg_gdba_create": (C.c_int, [C.POINTER(FgGdbaDesc), C.POINTER(P)]),
    "fg_gdba_destroy": (C.c_int, [P]),
    "fg_gdba_last_error": (C.c_char_p, [P]),
    "fg_gdba_init": (C.c_int, [P, P]),
    "fg_gdba_step": (C.c_int, [P, C.c_int32, P]),
    "fg_gdba_current": (C.c_int, [P, C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "fg_gdba_launch_count": (C.c_int64, [P]),
    "fg_dba_create": (C.c_int, [C.POINTER(FgDbaDesc), C.POINTER(P)]),
    "fg_dba_destroy": (C.c_int, [P]),
    "fg_dba_last_error": (C.c_char_p, [P]),
    "fg_dba_init": (C.c_int, [P, P]),
    "fg_dba_step": (C.c_int, [P, C.c_int32, P]),
    "fg_dba_current": (C.c_int, [P, C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "fg_dba_launch_count": (C.c_int64, [P]),
    "fg_syncbb_create": (C.c_int, [C.POINTER(FgSyncbbDesc), C.POINTER(P)]),
    "fg_syncbb_destroy": (C.c_int, [P]),
    "fg_syncbb_last_error": (C.c_char_p, [P]),
    "fg_syncbb_init": (C.c_int, [P, P]),
    "fg_syncbb_step": (C.c_int, [P, C.c_int64, P]),
    "fg_syncbb_current": (C.c_int, [P, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "fg_syncbb_launch_count": (C.c_int64, [P]),
    "fg_dpop_create": (C.c_int, [C.POINTER(FgDpopDesc), C.POINTER(P)]),
    "fg_dpop_destroy": (C.c_int, [P]),
    "fg_dpop_last_error": (C.c_char_p, [P]),
    "fg_dpop_run": (C.c_int, [P, P]),
    "fg_dpop_launch_count": (C.c_int64, [P]),
    "fg_mixeddsa_create": (C.c_int, [C.POINTER(FgMixedDsaDesc), C.POINTER(P)]),
    "fg_mixeddsa_destroy": (C.c_int, [P]),
    "fg_mixeddsa_last_error": (C.c_char_p, [P]),
    "fg_mixeddsa_init": (C.c_int, [P, P]),
    "fg_mixeddsa_step": (C.c_int, [P, C.c_int32, P]),
    "fg_mixeddsa_current": (C.c_int, [P, C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "fg_mixeddsa_launch_count": (C.c_int64, [P]),
    "fg_solution_cost": (C.c_int, [C.c_int32, C.c_int32, C.POINTER(FgClass), P, P, P, P, P,
                                   C.c_int32, P, P, C.c_double, P, P]),
    "fg_solution_cost_segmented": (C.c_int, [C.c_int32, C.c_int32, C.POINTER(FgClass), P, P, P, P, P,
                                             C.c_int32, P, P, P, P, C.c_int32, C.c_double, P, P]),
    "fg_gather_rows": (C.c_int, [C.c_int32, P, P, P, C.c_int64, C.c_int64, P]),
    "fg_trace_create": (C.c_int, [C.POINTER(FgTraceDesc), C.POINTER(P)]),
    "fg_trace_destroy": (C.c_int, [P]),
    "fg_trace_last_error": (C.c_char_p, [P]),
    "fg_trace_start": (C.c_int, [P, P]),
    "fg_trace_rows": (C.c_int, [P, C.POINTER(C.c_int64)]),
    "fg_trace_set_best": (C.c_int, [P, C.c_int32, P, P, P, P]),
    "fg_maxsum_set_trace": (C.c_int, [P, P]),
    "fg_dsa_set_trace": (C.c_int, [P, P]),
    "fg_mgm_set_trace": (C.c_int, [P, P]),
    "fg_mgm2_set_trace": (C.c_int, [P, P]),
    "fg_gdba_set_trace": (C.c_int, [P, P]),
    "fg_dba_set_trace": (C.c_int, [P, P]),
    "fg_mixeddsa_set_trace": (C.c_int, [P, P]),
}

_lib = None


class EngineError(RuntimeError):
    pass


def load():
    """Load libpydcop_b200.so and bind every declared symbol; raise if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EngineError(
            f"{LIB_PATH} is missing: build it with `python -m pydcop_b200.build` "
            "(pydcop_b200 has no CPU fallback for the MaxSum/DSA hot path)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    if lib.fg_abi_version() != FG_ABI_VERSION:
        raise EngineError("libpydcop_b200.so ABI version mismatch: rebuild it")
    _lib = lib
    return lib
