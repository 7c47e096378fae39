"""ctypes binding of the C-ABI in include/seist_b200.h (libseist_b200.so, built in-tree).

There is NO fallback: if the shared library is missing or its ABI does not match, importing the
compute path raises.  Build with `python __graft_entry__.py` (or `make -C seist_b200/csrc`).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libseist_b200.so")
ABI_VERSION = 24
MAX_IN = 3
MAX_WORLD = 8
SIG_LANES = 4


class SeistBN(C.Structure):
    _fields_ = [
        ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("running_mean", C.c_void_p), ("running_var", C.c_void_p),
        ("stat", C.c_void_p), ("gstat", C.c_void_p), ("stat_acc", C.c_void_p), ("gstat_acc", C.c_void_p),
        ("dgamma", C.c_void_p), ("dbeta", C.c_void_p), ("coef", C.c_void_p),
        ("count", C.c_double),
        ("C", C.c_int32), ("chain", C.c_int32), ("use_batch", C.c_int32), ("is_chained", C.c_int32),
        ("eps", C.c_float), ("momentum", C.c_float), ("grad_scale", C.c_float),
    ]


class SeistComm(C.Structure):
    _fields_ = [
        ("world", C.c_int32), ("rank", C.c_int32),
        ("stat_peer", C.c_void_p * MAX_WORLD), ("gstat_peer", C.c_void_p * MAX_WORLD),
        ("grad_peer", C.c_void_p * MAX_WORLD), ("sig_peer", C.c_void_p * MAX_WORLD),
        ("epoch", C.c_void_p), ("err", C.c_void_p),
    ]


class SeistView(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("g", C.c_void_p),
        ("Ct", C.c_int32), ("c0", C.c_int32), ("C", C.c_int32), ("L", C.c_int32),
        ("bn", C.c_int32), ("bn_c0", C.c_int32), ("act", C.c_int32), ("accum", C.c_int32),
    ]


class SeistOp(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("N", C.c_int32),
        ("bn_table", C.c_void_p), ("step_seed", C.c_void_p),
        ("inp", SeistView * MAX_IN),
        ("res_a", SeistView), ("res_b", SeistView), ("out", SeistView),
        ("out_dxd", C.c_void_p),
        ("W", C.c_void_p), ("bias", C.c_void_p), ("dW", C.c_void_p), ("dbias", C.c_void_p),
        ("n_in", C.c_int32), ("Cin", C.c_int32), ("Cout", C.c_int32), ("k", C.c_int32),
        ("stride", C.c_int32), ("pad_left", C.c_int32), ("groups", C.c_int32), ("pool", C.c_int32),
        ("up_src_L", C.c_int32), ("L_in", C.c_int32), ("L_out", C.c_int32), ("out_act", C.c_int32),
        ("out_scale", C.c_float),
        ("p_elem", C.c_float), ("p_path", C.c_float), ("p_alpha", C.c_float),
        ("seed_elem", C.c_uint32), ("seed_path", C.c_uint32), ("seed_alpha", C.c_uint32),
        ("lse", C.c_void_p), ("delta", C.c_void_p),
        ("heads", C.c_int32), ("p_attn", C.c_float), ("seed_attn", C.c_uint32), ("pad0_", C.c_int32),
        ("comm", C.c_void_p),
        ("zero_bytes", C.c_uint64), ("n_bn", C.c_int32), ("bn_lo", C.c_int32),
        ("lane", C.c_int32), ("n_wait", C.c_int32), ("wait_ev", C.c_int32 * 4), ("rec_event", C.c_int32), ("pad1_", C.c_int32),
    ]


class SeistAugCfg(C.Structure):
    _fields_ = [
        ("generate_noise_rate", C.c_double), ("add_event_rate", C.c_double), ("shift_event_rate", C.c_double),
        ("drop_channel_rate", C.c_double), ("scale_amplitude_rate", C.c_double),
        ("pre_emphasis_rate", C.c_double), ("add_noise_rate", C.c_double), ("add_gap_rate", C.c_double),
        ("coda_ratio", C.c_double), ("min_snr", C.c_double), ("p_position_ratio", C.c_double),
        ("pre_emphasis_ratio", C.c_float),
        ("in_samples", C.c_int32), ("min_event_gap", C.c_int32),
        ("max_event_num", C.c_int32), ("norm_mode", C.c_int32),
        ("mask_percent", C.c_int32), ("noise_percent", C.c_int32), ("window", C.c_int32),
    ]


class SeistStreamStep(C.Structure):
    _fields_ = [
        ("f0", C.c_int64), ("r0", C.c_int64), ("f1", C.c_int64), ("r1", C.c_int64),
        ("k0", C.c_int64), ("tail", C.c_int64), ("kr", C.c_int64),
        ("S", C.c_int32), ("C", C.c_int32), ("W", C.c_int32), ("P", C.c_int32),
        ("nk", C.c_int32), ("norm_mode", C.c_int32), ("stack_mode", C.c_int32), ("pad_", C.c_int32),
    ]


class SeistRaggedStep(C.Structure):
    _fields_ = [
        ("f0", C.c_void_p), ("r0", C.c_void_p), ("f1", C.c_void_p), ("r1", C.c_void_p),
        ("k0", C.c_void_p), ("nk", C.c_void_p), ("tail", C.c_void_p), ("kr", C.c_void_p),
        ("win_off", C.c_void_p), ("chunk_off", C.c_void_p), ("acc_off", C.c_void_p), ("out_off", C.c_void_p),
        ("n_win", C.c_int64), ("max_len", C.c_int64),
        ("S", C.c_int32), ("C", C.c_int32), ("W", C.c_int32), ("P", C.c_int32),
        ("norm_mode", C.c_int32), ("stack_mode", C.c_int32),
    ]


# op kinds (enum SeistOpKind)
CONV_FWD, CONV_BWD_DATA, CONV_BWD_W, RES_BWD = 1, 2, 3, 4
ATT_FWD, ATT_BWD_Q, ATT_BWD_KV = 5, 6, 7
HEADVEC_FWD, HEADVEC_BWD = 8, 9
BN_FINALIZE_FWD, BN_FINALIZE_BWD, ZERO = 10, 11, 12
BN_PREPARE_FWD, BN_PREPARE_BWD = 13, 14
STEM_COMPOSE_FWD, STEM_COMPOSE_BWD = 15, 16

_lib = None


def lib():
    """Load (once) and return the shared library; raises if it is absent or mismatched."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise RuntimeError(
            f"seist_b200: CUDA extension not built ({LIB_PATH} missing). "
            "Run `python __graft_entry__.py` — there is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    L.seist_abi_version.restype = C.c_int
    L.seist_sizeof_op.restype = C.c_uint64
    L.seist_sizeof_bn.restype = C.c_uint64
    L.seist_last_error.restype = C.c_char_p
    L.seist_launch_count.restype = C.c_uint64
    L.seist_tc_error_flag.restype = C.c_int
    L.seist_op_family.restype = C.c_char_p
    L.seist_op_family.argtypes = [C.c_void_p]
    L.seist_plan_run.restype = C.c_int
    L.seist_plan_run.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    L.seist_plan_run_lanes.restype = C.c_int
    L.seist_plan_run_lanes.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32]
    L.seist_bce_fwd.restype = C.c_int
    L.seist_bce_fwd.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int64,
                                C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    L.seist_bce_bwd.restype = C.c_int
    L.seist_bce_bwd.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                C.c_int64, C.c_float, C.c_void_p, C.c_void_p]
    L.seist_ce_fwd.restype = C.c_int
    L.seist_ce_fwd.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_void_p, C.c_void_p,
                               C.c_void_p]
    L.seist_ce_bwd.restype = C.c_int
    L.seist_ce_bwd.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_void_p,
                               C.c_void_p]
    L.seist_huber_fwd.restype = C.c_int
    L.seist_huber_fwd.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p, C.c_void_p,
                                  C.c_void_p]
    L.seist_huber_bwd.restype = C.c_int
    L.seist_huber_bwd.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p,
                                  C.c_void_p]
    L.seist_adam_step.restype = C.c_int
    L.seist_adam_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                  C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int32,
                                  C.c_float, C.c_void_p]
    L.seist_sgd_step.restype = C.c_int
    L.seist_sgd_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_double,
                                 C.c_double, C.c_double, C.c_int32, C.c_float, C.c_void_p]
    L.seist_advance_seed.restype = C.c_int
    L.seist_advance_seed.argtypes = [C.c_void_p, C.c_void_p]
    L.seist_pick_phase.restype = C.c_int
    L.seist_pick_phase.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_int32,
                                   C.c_int64, C.c_void_p, C.c_void_p]
    L.seist_detect_event.restype = C.c_int
    L.seist_detect_event.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_int32,
                                     C.c_void_p, C.c_void_p]
    L.seist_pick_counters.restype = C.c_int
    L.seist_pick_counters.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    L.seist_det_counters.restype = C.c_int
    L.seist_det_counters.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                     C.c_void_p]
    L.seist_normalize.restype = C.c_int
    L.seist_normalize.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p]
    L.seist_dpk_labels.restype = C.c_int
    L.seist_dpk_labels.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_double, C.c_void_p, C.c_void_p]
    L.seist_sizeof_aug.restype = C.c_uint64
    L.seist_aug_recipe_bytes.restype = C.c_int
    L.seist_augment.restype = C.c_int
    L.seist_augment.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(SeistAugCfg), C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    L.seist_window_batch.restype = C.c_int
    L.seist_window_batch.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.c_int64, C.c_int32,
                                     C.c_int32, C.c_void_p, C.c_void_p]
    L.seist_event_windows.restype = C.c_int
    L.seist_event_windows.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                      C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
    L.seist_stack_batch.restype = C.c_int
    L.seist_stack_batch.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int32,
                                    C.c_void_p, C.c_void_p]
    L.seist_stack_finish.restype = C.c_int
    L.seist_stack_finish.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.c_void_p]
    L.seist_peaks_work_bytes.restype = C.c_int64
    L.seist_peaks_work_bytes.argtypes = [C.c_int32, C.c_int64]
    L.seist_peaks_long.restype = C.c_int
    L.seist_peaks_long.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_float, C.c_int32, C.c_void_p,
                                   C.c_int64, C.c_void_p, C.c_void_p]
    L.seist_peaks_long_fill.restype = C.c_int
    L.seist_peaks_long_fill.argtypes = [C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p]
    L.seist_runs_work_bytes.restype = C.c_int64
    L.seist_runs_work_bytes.argtypes = [C.c_int32, C.c_int64]
    L.seist_runs_long.restype = C.c_int
    L.seist_runs_long.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_float, C.c_void_p, C.c_int64,
                                  C.c_void_p, C.c_void_p]
    L.seist_runs_long_fill.restype = C.c_int
    L.seist_runs_long_fill.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_float, C.c_void_p,
                                       C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    step = C.POINTER(SeistStreamStep)
    L.seist_sizeof_stream_step.restype = C.c_uint64
    L.seist_stream_window.restype = C.c_int
    L.seist_stream_window.argtypes = [step, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]
    L.seist_stream_stack.restype = C.c_int
    L.seist_stream_stack.argtypes = [step, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.seist_stream_emit.restype = C.c_int
    L.seist_stream_emit.argtypes = [step, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.seist_stream_keep.restype = C.c_int
    L.seist_stream_keep.argtypes = [step, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.seist_stream_peaks_work_bytes.restype = C.c_int64
    L.seist_stream_peaks_work_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int64]
    rstep = C.POINTER(SeistRaggedStep)
    P, I32, I64, F32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    L.seist_sizeof_ragged_step.restype = C.c_uint64
    L.seist_ragged_window.restype = C.c_int
    L.seist_ragged_window.argtypes = [rstep, P, P, I64, I32, P, P]
    L.seist_ragged_stack.restype = C.c_int
    L.seist_ragged_stack.argtypes = [rstep, P, I64, I32, I32, I32, P, P, P]
    L.seist_ragged_emit.restype = C.c_int
    L.seist_ragged_emit.argtypes = [rstep, P, P, P, P, P]
    L.seist_ragged_keep.restype = C.c_int
    L.seist_ragged_keep.argtypes = [rstep, P, P, P, P]
    L.seist_ragged_ext.restype = C.c_int
    L.seist_ragged_ext.argtypes = [P, P, P, P, I32, I32, I64, P, P, P]
    L.seist_ragged_peaks.restype = C.c_int
    L.seist_ragged_peaks.argtypes = [P, P, I32, I32, I32, I64, P, P, I64, F32, I32, P, P, P, P, I32, P, I32, I64, P, I32, P, P, P]
    L.seist_ragged_peaks_fill.restype = C.c_int
    L.seist_ragged_peaks_fill.argtypes = [I32, I64, P, I32, P, P, P, P, P]
    L.seist_ragged_runs.restype = C.c_int
    L.seist_ragged_runs.argtypes = [P, P, I32, I32, I32, I64, P, P, I64, F32, P, P, P, I64, P, P]
    L.seist_ragged_runs_fill.restype = C.c_int
    L.seist_ragged_runs_fill.argtypes = [P, P, I32, I32, I32, I64, P, P, I64, F32, P, P, P, P, I64, P, P, P]
    L.seist_ragged_history.restype = C.c_int
    L.seist_ragged_history.argtypes = [P, P, P, I64, P, P, I64, P, P, I32, I32, I64, P, I64, P]
    L.seist_ragged_event_windows.restype = C.c_int
    L.seist_ragged_event_windows.argtypes = [P, P, P, I64, I32, I32, P, I64, P, I64, I32, I32, I32, I32, P, I32, P]
    L.seist_gap_event_windows.restype = C.c_int
    L.seist_gap_event_windows.argtypes = [P, P, P, I64, I32, I32, P, P, P, P, I32, P, I64, I64, I32, I32, I32, I32, P, I32, P]
    L.seist_gap_segments.restype = C.c_int
    L.seist_gap_segments.argtypes = [P, I32, I32, I64, P, I64, P, P]
    L.seist_gap_segments_fill.restype = C.c_int
    L.seist_gap_segments_fill.argtypes = [P, I32, I32, I64, P, I64, P, P, I64, P]
    L.seist_segment_window.restype = C.c_int
    L.seist_segment_window.argtypes = [P, I32, I32, I64, P, P, P, I32, I64, I32, I32, I64, I32, I32, P, P]
    L.seist_segment_stack.restype = C.c_int
    L.seist_segment_stack.argtypes = [P, I32, I64, P, P, P, I32, I64, I32, I32, I64, I32, I32, I32, I32, P, P]
    L.seist_segment_finish.restype = C.c_int
    L.seist_segment_finish.argtypes = [P, I32, I64, P, P, I32, I32, I32, I32, P]
    L.seist_segment_gather.restype = C.c_int
    L.seist_segment_gather.argtypes = [P, I32, I64, P, P, I32, P, P, I32, I64, P, I64, P]
    L.seist_segment_event_windows.restype = C.c_int
    L.seist_segment_event_windows.argtypes = [P, I32, I32, I64, P, P, P, I32, P, I64, P, I64, I32, I32, I32, I32, P, I32, P]
    L.seist_gap_stream_scan.restype = C.c_int
    L.seist_gap_stream_scan.argtypes = [P, I64, P, I32, I32, I64, P, I64, P, P]
    L.seist_gap_stream_fill.restype = C.c_int
    L.seist_gap_stream_fill.argtypes = [P, I64, P, I32, I32, I64, P, I64, P, P, I64, P]
    L.seist_gap_stream_pack.restype = C.c_int
    L.seist_gap_stream_pack.argtypes = [P, I64, P, I32, I32, P, P, P, I32, I64, P, I64, P]
    L.seist_gap_stream_copy.restype = C.c_int
    L.seist_gap_stream_copy.argtypes = [P, I64, P, P, P, P, P, I32, I64, P, I64, P]
    L.seist_resample.restype = C.c_int
    L.seist_resample.argtypes = [P, I32, I64, P, I32, I32, P, P]
    L.seist_resample_stream.restype = C.c_int
    L.seist_resample_stream.argtypes = [P, I64, P, I64, P, I32, I32, I64, P, I32, I32, P, I64, P, P]
    L.seist_resample_table.restype = C.c_int
    L.seist_resample_table.argtypes = [I32, P, P, P]
    L.seist_resample_multi.restype = C.c_int
    L.seist_resample_multi.argtypes = [P, I32, I32, I64, I64, P, I32, I32, P, P, P]
    L.seist_resample_multi_stream.restype = C.c_int
    L.seist_resample_multi_stream.argtypes = [P, I64, P, I64, P, I32, I32, I64, P, I32, I32, P, P, I64, P, P]
    L.seist_sizeof_comm.restype = C.c_uint64
    L.seist_comm_barrier.restype = C.c_int
    L.seist_comm_barrier.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
    L.seist_comm_allreduce.restype = C.c_int
    L.seist_comm_allreduce.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]
    if L.seist_abi_version() != ABI_VERSION:
        raise RuntimeError(f"seist_b200: ABI mismatch (lib {L.seist_abi_version()} != {ABI_VERSION})")
    if L.seist_sizeof_op() != C.sizeof(SeistOp) or L.seist_sizeof_bn() != C.sizeof(SeistBN):
        raise RuntimeError(
            f"seist_b200: struct layout mismatch op {L.seist_sizeof_op()} vs {C.sizeof(SeistOp)}, "
            f"bn {L.seist_sizeof_bn()} vs {C.sizeof(SeistBN)}")
    if L.seist_sizeof_comm() != C.sizeof(SeistComm):
        raise RuntimeError(f"seist_b200: SeistComm layout mismatch {L.seist_sizeof_comm()} vs {C.sizeof(SeistComm)}")
    if L.seist_sizeof_aug() != C.sizeof(SeistAugCfg):
        raise RuntimeError(f"seist_b200: SeistAugCfg layout mismatch {L.seist_sizeof_aug()} vs {C.sizeof(SeistAugCfg)}")
    if L.seist_sizeof_stream_step() != C.sizeof(SeistStreamStep):
        raise RuntimeError(f"seist_b200: SeistStreamStep layout mismatch {L.seist_sizeof_stream_step()} vs {C.sizeof(SeistStreamStep)}")
    if L.seist_sizeof_ragged_step() != C.sizeof(SeistRaggedStep):
        raise RuntimeError(f"seist_b200: SeistRaggedStep layout mismatch {L.seist_sizeof_ragged_step()} vs {C.sizeof(SeistRaggedStep)}")
    _lib = L
    return L


EXPORTS = [
    "seist_abi_version", "seist_sizeof_op", "seist_sizeof_bn", "seist_last_error", "seist_launch_count",
    "seist_tc_error_flag", "seist_plan_run", "seist_plan_run_lanes", "seist_bce_fwd", "seist_bce_bwd", "seist_huber_fwd", "seist_huber_bwd",
    "seist_adam_step", "seist_sgd_step", "seist_advance_seed", "seist_comm_allreduce", "seist_comm_barrier", "seist_sizeof_comm", "seist_op_family",
    "seist_pick_phase", "seist_detect_event", "seist_pick_counters", "seist_det_counters",
    "seist_normalize", "seist_dpk_labels", "seist_ce_fwd", "seist_ce_bwd",
    "seist_augment", "seist_sizeof_aug", "seist_aug_recipe_bytes",
    "seist_window_batch", "seist_event_windows", "seist_stack_batch", "seist_stack_finish", "seist_peaks_work_bytes", "seist_peaks_long",
    "seist_peaks_long_fill", "seist_runs_work_bytes", "seist_runs_long", "seist_runs_long_fill",
    "seist_sizeof_stream_step", "seist_stream_window", "seist_stream_stack", "seist_stream_emit", "seist_stream_keep",
    "seist_stream_peaks_work_bytes",
    "seist_sizeof_ragged_step", "seist_ragged_window", "seist_ragged_stack", "seist_ragged_emit", "seist_ragged_keep", "seist_ragged_ext",
    "seist_ragged_peaks", "seist_ragged_peaks_fill", "seist_ragged_runs", "seist_ragged_runs_fill",
    "seist_ragged_history", "seist_ragged_event_windows",
    "seist_gap_segments", "seist_gap_segments_fill", "seist_segment_window", "seist_segment_stack", "seist_segment_finish",
    "seist_segment_gather", "seist_segment_event_windows",
    "seist_gap_stream_scan", "seist_gap_stream_fill", "seist_gap_stream_pack", "seist_gap_stream_copy",
    "seist_gap_event_windows",
    "seist_resample", "seist_resample_stream", "seist_resample_table", "seist_resample_multi", "seist_resample_multi_stream",
]


def check(rc: int, what: str = "seist"):
    if rc != 0:
        msg = lib().seist_last_error()
        raise RuntimeError(f"{what} failed: status {rc}: {msg.decode() if msg else ''}")
