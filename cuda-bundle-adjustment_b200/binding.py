"""ctypes binding of libcuba_b200.so (include/cuba_b200.h).  Mirrors the reference's operator interface
for the hot path: initialize()/optimize(n)/batchStatistics()/timeProfile()/chiSquared()
(reference include/cuda_bundle_adjustment.h:34-125) on a flat problem."""
import ctypes as C
import dataclasses
import os

import numpy as np

from . import graphio

HERE = os.path.dirname(os.path.abspath(__file__))
ROBUST_NONE, ROBUST_HUBER, ROBUST_TUKEY = 0, 1, 2
EDGE_MONOCULAR, EDGE_STEREO = 0, 1
# reference src/cuda_bundle_adjustment.cpp:547-557
PROFILE_ITEMS = ("0: Initialize Optimizer", "1: Build Structure", "2: Compute Error", "3: Build System",
                 "4: Schur Complement", "5: Symbolic Decomposition", "6: Numerical Decomposition", "7: Update Solution")


# cuba_debug_get_pcg_info (include/cuba_b200.h): info[] fields and the kernel names behind CUBA_PCG_KERNEL_* / CUBA_COARSE_KERNEL_*
PCG_INFO_LEN = 16
PCG_INFO_FIELDS = ("kernel", "two_level", "aggs_per_cta", "G", "gs", "A", "maxRows", "capBlocks", "zhInSmem", "coarse_kernel",
                   "cinfo", "status", "iters", "coarse_rebuilds", "bj_retries", "bad_rebuilds")
PCG_KERNELS = ("none", "k_pcg", "k_pcg2", "k_pcg3", "k_pcg4", "k_pcg5", "k_pcg5_big", "k_pcg5t", "k_dense_chol")   # "k_pcg" (retired) is never reported
COARSE_KERNELS = ("none", "k_coarse_invert", "cluster2<8>", "cluster2<16>", "k_coarse_dense", "k_coarse_chol_cluster")   # the cluster kernels (retired) are never reported


# cuba_debug_pcg5_plan: info[] fields; w_cols_tuned / w_cols_legacy are the columns of w each launch shape's staging holds
PCG5_PLAN_FIELDS = ("ok", "G", "gs", "A", "needMax", "maxRows", "maxNeedAgg", "halo_rows", "blkMax", "w_cols_tuned", "w_cols_legacy")


class CubaError(RuntimeError):
    pass


# the status word of the device-resident batches (include/cuba_b200.h: CUBA_BATCH_*): a bit per failed check
BATCH_STATUS = {1: "ptr does not start at 0", 2: "ptr decreases", 4: "ptr does not end at the item count",
                8: "non-finite omega or pair value", 16: "non-finite S12 or intrinsics", 32: "s <= 0", 64: "iP outside [0, P)"}


ITER_STAT_DTYPE = np.dtype([("iteration", "<i4"), ("trials", "<i4"), ("chi2", "<f8"), ("lambda_", "<f8"), ("pcg_iters", "<i4"),
                            ("pcg_failed", "<i4")])


def stats_view(stats):
    """the stats tensor of optimize_poses_device / optimize_sim3_device / optimize_points_device ([B, S, 4] float64 words) as the
    structured [B, S] array the _flat methods return; copies to the host, so it waits for the call"""
    a = np.ascontiguousarray(stats.cpu().numpy())
    return a.view(ITER_STAT_DTYPE).reshape(a.shape[:2])


def batch_status_message(status):
    """the checks a status word of optimize_poses_device / optimize_sim3_device / optimize_points_device reports as failed, as text
    ("ok" for 0)"""
    status = int(status)
    return "; ".join(m for bit, m in BATCH_STATUS.items() if status & bit) or ("ok" if status == 0 else "unknown status %d" % status)


def library_path():
    return os.path.join(HERE, "libcuba_b200.so")


class _Config(C.Structure):
    _fields_ = [("device", C.c_int), ("use_fp32", C.c_int), ("pcg_max_iters", C.c_int), ("pcg_tol", C.c_double),
                ("deterministic", C.c_int), ("reserved", C.c_int * 7)]


class _Problem(C.Structure):
    _fields_ = [("Pall", C.c_int32), ("numP", C.c_int32), ("Lall", C.c_int32), ("numL", C.c_int32),
                ("q", C.c_void_p), ("t", C.c_void_p), ("cam", C.c_void_p), ("Xw", C.c_void_p),
                ("E2", C.c_int32), ("idx2", C.c_void_p), ("meas2", C.c_void_p), ("omega2", C.c_void_p),
                ("E3", C.c_int32), ("idx3", C.c_void_p), ("meas3", C.c_void_p), ("omega3", C.c_void_p)]


class _IterStat(C.Structure):
    _fields_ = [("iteration", C.c_int32), ("trials", C.c_int32), ("chi2", C.c_double), ("lambda_", C.c_double),
                ("pcg_iters", C.c_int32), ("pcg_failed", C.c_int32)]


class _Sizes(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("Pall", "numP", "Lall", "numL", "E2", "E3", "nhpl", "nblk", "nmul", "nblk_full")]


class _PoseBatch(C.Structure):
    _fields_ = [("B", C.c_int32), ("E2", C.c_int32), ("E3", C.c_int32), ("q", C.c_void_p), ("t", C.c_void_p), ("cam", C.c_void_p),
                ("ptr2", C.c_void_p), ("X2", C.c_void_p), ("meas2", C.c_void_p), ("omega2", C.c_void_p),
                ("ptr3", C.c_void_p), ("X3", C.c_void_p), ("meas3", C.c_void_p), ("omega3", C.c_void_p)]


class _PoseRound(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("kernel_type", C.c_int32 * 2), ("delta", C.c_double * 2), ("restart", C.c_int32),
                ("chi2_mono", C.c_double), ("chi2_stereo", C.c_double), ("flags", C.c_int32)]


POSE_MAX_ROUNDS = 8      # CUBA_POSE_MAX_ROUNDS


@dataclasses.dataclass
class PoseRound:
    """One round of Engine.optimize_poses (include/cuba_b200.h: cuba_pose_round): optimize(iterations) under kernel / delta
    (mono, stereo), from the frame's input pose when restart is set, then the outlier test of classify_edges on the result."""
    iterations: int = 10
    kernel: tuple = (ROBUST_NONE, ROBUST_NONE)
    delta: tuple = (0.0, 0.0)
    restart: bool = True
    chi2_mono: float = 5.991
    chi2_stereo: float = 7.815
    depth: bool = False
    reinclude: bool = True


def orbslam2_pose_schedule():
    """ORB-SLAM2's Optimizer::PoseOptimization: four rounds of optimize(10) from the frame's pose, Huber in the first two, the chi2
    test with re-inclusion after each"""
    huber = dict(kernel=(ROBUST_HUBER, ROBUST_HUBER), delta=(5.991 ** 0.5, 7.815 ** 0.5))
    return [PoseRound(**(huber if r < 2 else {})) for r in range(4)]


class _PointBatch(C.Structure):
    _fields_ = [("B", C.c_int32), ("P", C.c_int32), ("E2", C.c_int32), ("E3", C.c_int32), ("Xw", C.c_void_p), ("q", C.c_void_p),
                ("t", C.c_void_p), ("cam", C.c_void_p), ("ptr2", C.c_void_p), ("iP2", C.c_void_p), ("meas2", C.c_void_p),
                ("omega2", C.c_void_p), ("ptr3", C.c_void_p), ("iP3", C.c_void_p), ("meas3", C.c_void_p), ("omega3", C.c_void_p)]


class _Sim3Batch(C.Structure):
    _fields_ = [("B", C.c_int32), ("N", C.c_int32), ("ptr", C.c_void_p), ("q", C.c_void_p), ("t", C.c_void_p), ("s", C.c_void_p),
                ("cam1", C.c_void_p), ("cam2", C.c_void_p), ("fix_scale", C.c_void_p), ("X1", C.c_void_p), ("X2", C.c_void_p),
                ("obs1", C.c_void_p), ("obs2", C.c_void_p), ("omega1", C.c_void_p), ("omega2", C.c_void_p)]


class _Sim3Params(C.Structure):
    _fields_ = [("chi2", C.c_double), ("iterations", C.c_int32), ("iterations_bad", C.c_int32), ("iterations_good", C.c_int32),
                ("min_pairs", C.c_int32)]


@dataclasses.dataclass
class Sim3Params:
    """OptimizeSim3's schedule (include/cuba_b200.h: cuba_sim3_params), ORB-SLAM2's values by default: optimize(iterations), the pair
    test at chi2 (also the square of the Huber delta), then, with at least min_pairs pairs left, optimize(iterations_bad) if the test
    removed a pair, else optimize(iterations_good), and the test again."""
    chi2: float = 10.0
    iterations: int = 5
    iterations_bad: int = 10
    iterations_good: int = 5
    min_pairs: int = 10


_lib = None

_SYMBOLS = [
    "cuba_last_error", "cuba_version", "cuba_engine_create", "cuba_engine_destroy", "cuba_engine_set_robust_kernel",
    "cuba_comm_unique_id", "cuba_engine_set_comm", "cuba_engine_set_problem", "cuba_engine_set_linear_solver", "cuba_engine_set_structure_reuse", "cuba_engine_get_structure_reuses", "cuba_engine_set_state", "cuba_engine_get_sizes", "cuba_engine_reset_state", "cuba_engine_get_stream", "cuba_engine_get_device", "cuba_engine_flush_l2",
    "cuba_engine_optimize", "cuba_engine_get_state", "cuba_engine_get_chi2", "cuba_engine_set_edge_levels", "cuba_engine_get_edge_levels", "cuba_engine_classify_edges", "cuba_engine_set_problem_device", "cuba_engine_set_state_device", "cuba_engine_get_state_device", "cuba_engine_get_chi2_device", "cuba_engine_set_edge_levels_device", "cuba_engine_get_edge_levels_device", "cuba_engine_optimize_poses", "cuba_engine_optimize_sim3", "cuba_pose_batch_workspace_bytes", "cuba_engine_optimize_poses_device", "cuba_sim3_batch_workspace_bytes", "cuba_engine_optimize_sim3_device", "cuba_engine_optimize_points", "cuba_point_batch_workspace_bytes", "cuba_engine_optimize_points_device", "cuba_engine_optimize_landmarks", "cuba_engine_optimize_landmarks_device", "cuba_engine_get_profile",
    "cuba_engine_get_launch_count", "cuba_get_transfer_bytes", "cuba_stage_linearize", "cuba_stage_max_diagonal", "cuba_stage_solve", "cuba_stage_update",
    "cuba_stage_commit", "cuba_stage_chi2", "cuba_debug_get_hpl_structure", "cuba_debug_get_hsc_structure",
    "cuba_debug_get_system", "cuba_debug_get_schur", "cuba_debug_get_delta", "cuba_debug_get_pcg_info", "cuba_debug_get_coarse", "cuba_debug_coarse_inverse", "cuba_debug_dense_solve", "cuba_debug_peer_allreduce", "cuba_debug_pcg5_ranks", "cuba_debug_build_structure_host", "cuba_debug_pcg_partition", "cuba_debug_pcg5_plan", "cuba_debug_pcg5_plan_apc", "cuba_debug_pcg5t_layout", "cuba_debug_dense_layout", "cuba_debug_dropin_problem", "cuba_debug_dropin_levels", "cuba_bench_stage",
]


def exported_symbols():
    return list(_SYMBOLS)


def load_library():
    """Loads the in-tree libcuba_b200.so; raises (never falls back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        raise CubaError("%s not built: run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)" % path)
    L = C.CDLL(path)
    L.cuba_last_error.restype = C.c_char_p
    vp, i, d = C.c_void_p, C.c_int, C.c_double
    sig = {
        "cuba_engine_create": [C.POINTER(_Config), C.POINTER(vp)],
        "cuba_engine_destroy": [vp],
        "cuba_engine_set_robust_kernel": [vp, i, i, d],
        "cuba_comm_unique_id": [vp],
        "cuba_engine_set_comm": [vp, i, i, vp],
        "cuba_engine_set_problem": [vp, C.POINTER(_Problem)],
        "cuba_engine_set_linear_solver": [vp, i],
        "cuba_engine_set_structure_reuse": [vp, i],
        "cuba_engine_get_structure_reuses": [vp, C.POINTER(C.c_longlong)],
        "cuba_engine_set_state": [vp, vp, vp, vp],
        "cuba_engine_get_sizes": [vp, C.POINTER(_Sizes)],
        "cuba_engine_reset_state": [vp],
        "cuba_engine_get_stream": [vp, C.POINTER(vp)],
        "cuba_engine_get_device": [vp, C.POINTER(i)],
        "cuba_engine_flush_l2": [vp],
        "cuba_engine_optimize": [vp, i, vp, C.POINTER(i)],
        "cuba_engine_get_state": [vp, vp, vp, vp],
        "cuba_engine_get_chi2": [vp, vp],
        "cuba_engine_set_edge_levels": [vp, vp],
        "cuba_engine_get_edge_levels": [vp, vp],
        "cuba_engine_classify_edges": [vp, d, d, i, vp],
        "cuba_engine_set_problem_device": [vp, C.POINTER(_Problem), vp],
        "cuba_engine_set_state_device": [vp, vp, vp, vp, vp],
        "cuba_engine_get_state_device": [vp, vp, vp, vp, vp],
        "cuba_engine_get_chi2_device": [vp, vp, vp],
        "cuba_engine_set_edge_levels_device": [vp, vp, vp],
        "cuba_engine_get_edge_levels_device": [vp, vp, vp],
        "cuba_engine_optimize_poses": [vp, C.POINTER(_PoseBatch), i, vp, vp, vp, vp, vp, vp, vp],
        "cuba_engine_optimize_sim3": [vp, C.POINTER(_Sim3Batch), C.POINTER(_Sim3Params), vp, vp, vp, vp, vp, vp, vp],
        "cuba_engine_optimize_poses_device": [vp, C.POINTER(_PoseBatch), i, vp, vp, C.c_size_t, vp, vp, vp, vp, vp, vp, vp, vp],
        "cuba_engine_optimize_sim3_device": [vp, C.POINTER(_Sim3Batch), C.POINTER(_Sim3Params), vp, C.c_size_t, vp, vp, vp, vp, vp, vp, vp,
                                             vp, vp],
        "cuba_engine_optimize_points": [vp, C.POINTER(_PointBatch), i, vp, vp, vp, vp, vp, vp],
        "cuba_engine_optimize_points_device": [vp, C.POINTER(_PointBatch), i, vp, vp, C.c_size_t, vp, vp, vp, vp, vp, vp, vp],
        "cuba_engine_optimize_landmarks": [vp, vp, C.c_int32, i, vp, vp, vp, vp],
        "cuba_engine_optimize_landmarks_device": [vp, vp, C.c_int32, i, vp, vp, vp, vp, vp],
        "cuba_engine_get_profile": [vp, vp],
        "cuba_engine_get_launch_count": [vp, C.POINTER(C.c_longlong)],
        "cuba_get_transfer_bytes": [C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)],
        "cuba_stage_linearize": [vp, C.POINTER(d)],
        "cuba_stage_max_diagonal": [vp, C.POINTER(d)],
        "cuba_stage_solve": [vp, d, C.POINTER(i), C.POINTER(i)],
        "cuba_stage_update": [vp, d, C.POINTER(d), C.POINTER(d)],
        "cuba_stage_commit": [vp, i],
        "cuba_stage_chi2": [vp, C.POINTER(d)],
        "cuba_debug_get_hpl_structure": [vp, vp, vp, vp],
        "cuba_debug_get_hsc_structure": [vp, vp, vp],
        "cuba_debug_get_system": [vp, vp, vp, vp, vp, vp],
        "cuba_debug_get_schur": [vp, vp, vp, vp],
        "cuba_debug_get_delta": [vp, vp, vp],
        "cuba_debug_get_pcg_info": [vp, vp, C.POINTER(d)],
        "cuba_debug_get_coarse": [vp, vp, vp, vp],
        "cuba_debug_coarse_inverse": [vp, vp, i, vp, vp],
        "cuba_debug_dense_solve": [vp, vp, vp, i, vp, C.POINTER(i)],
        "cuba_debug_peer_allreduce": [vp, i, C.c_int64, i, vp, vp],
        "cuba_debug_pcg5_ranks": [vp, i, i, i, vp, vp, vp, vp, vp],
        "cuba_debug_build_structure_host": [C.POINTER(_Problem), i, i, C.POINTER(_Sizes), vp, vp, vp, vp, vp, vp, vp, vp],
        "cuba_debug_pcg_partition": [C.POINTER(_Problem), i, i, vp],
        "cuba_debug_pcg5_plan": [C.POINTER(_Problem), i, i, i, vp],
        "cuba_debug_pcg5_plan_apc": [C.POINTER(_Problem), i, i, i, i, vp, C.POINTER(C.c_uint64)],
        "cuba_debug_pcg5t_layout": [C.POINTER(_Problem), i, i, i, C.c_int64, vp],
        "cuba_debug_dense_layout": [C.POINTER(_Problem), vp, vp],
        "cuba_debug_dropin_problem": [vp, C.POINTER(_Problem)],
        "cuba_debug_dropin_levels": [vp, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_int32)],
        "cuba_bench_stage": [vp, i, i, i, d, C.POINTER(d)],
    }
    for name, args in sig.items():
        fn = getattr(L, name)
        fn.argtypes = args
        fn.restype = C.c_int
    L.cuba_pose_batch_workspace_bytes.argtypes = [i, i, i, i, vp, i]
    L.cuba_pose_batch_workspace_bytes.restype = C.c_size_t
    L.cuba_sim3_batch_workspace_bytes.argtypes = [i, i, C.POINTER(_Sim3Params), i]
    L.cuba_sim3_batch_workspace_bytes.restype = C.c_size_t
    L.cuba_point_batch_workspace_bytes.argtypes = [i, i, i, i, i, vp, i]
    L.cuba_point_batch_workspace_bytes.restype = C.c_size_t
    _lib = L
    return L


def _check(rc):
    if rc != 0:
        raise CubaError("cuba error %d: %s" % (rc, load_library().cuba_last_error().decode()))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _dp(a):
    return None if a is None else a.data_ptr()


def _f64(a, w):
    """a as a contiguous float64 array [n, w] ([n] for w = 1)"""
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape((-1, w) if w > 1 else (-1,)))


def _problem_struct(prob):
    keep = [np.ascontiguousarray(prob.q, dtype=np.float64), np.ascontiguousarray(prob.t, dtype=np.float64),
            np.ascontiguousarray(prob.cam, dtype=np.float64), np.ascontiguousarray(prob.Xw, dtype=np.float64),
            np.ascontiguousarray(prob.idx2, dtype=np.int32), np.ascontiguousarray(prob.meas2, dtype=np.float64),
            np.ascontiguousarray(prob.omega2, dtype=np.float64), np.ascontiguousarray(prob.idx3, dtype=np.int32),
            np.ascontiguousarray(prob.meas3, dtype=np.float64), np.ascontiguousarray(prob.omega3, dtype=np.float64)]
    P = _Problem(prob.Pall, prob.numP, prob.Lall, prob.numL, _p(keep[0]), _p(keep[1]), _p(keep[2]), _p(keep[3]),
                 prob.E2, _p(keep[4]), _p(keep[5]), _p(keep[6]), prob.E3, _p(keep[7]), _p(keep[8]), _p(keep[9]))
    return P, keep


def transfer_bytes():
    """(h2d, d2h) bytes copied so far by this thread's engines"""
    a, b = C.c_longlong(0), C.c_longlong(0)
    _check(load_library().cuba_get_transfer_bytes(C.byref(a), C.byref(b)))
    return a.value, b.value


def build_structure_host(prob, rank=0, world=1):
    """Host-only structure build (no GPU needed): dict of index arrays + sizes."""
    L = load_library()
    P, keep = _problem_struct(prob)
    sz = _Sizes()
    _check(L.cuba_debug_build_structure_host(C.byref(P), rank, world, C.byref(sz), None, None, None, None, None, None, None, None))
    out = {n: getattr(sz, n) for n, _ in _Sizes._fields_}
    arrs = {"hplColPtr": np.zeros(sz.numL + 1, np.int32), "hplRowInd": np.zeros(sz.nhpl, np.int32),
            "edge2Hpl": np.zeros(sz.E2 + sz.E3, np.int32), "hscRowPtr": np.zeros(sz.numP + 1, np.int32),
            "hscColInd": np.zeros(sz.nblk, np.int32), "fullRowPtr": np.zeros(sz.numP + 1, np.int32),
            "fullColInd": np.zeros(sz.nblk_full, np.int32), "shard": np.zeros(4, np.int32)}
    _check(L.cuba_debug_build_structure_host(C.byref(P), rank, world, C.byref(sz), *[_p(arrs[k]) for k in
           ("hplColPtr", "hplRowInd", "edge2Hpl", "hscRowPtr", "hscColInd", "fullRowPtr", "fullColInd", "shard")]))
    out.update(arrs)
    return out


def pcg_partition_host(prob, n_ctas=148, max_aggregates=74):
    """Host side of the PCG setup on the CPU (row partition over n_ctas persistent CTAs, need lists, pose aggregates and coarse
    lists of the two-level PCG); the library verifies their invariants and raises CubaError if one fails."""
    L = load_library()
    P, keep = _problem_struct(prob)
    info = np.zeros(9, np.int32)
    _check(L.cuba_debug_pcg_partition(C.byref(P), int(n_ctas), int(max_aggregates), _p(info)))
    return dict(zip(("G", "gs", "A", "needMax", "maxRows", "blkMax", "maxNeedAgg", "coarse_list_size", "pcg3_fixed_bytes"), (int(v) for v in info)))


def pcg5_plan_host(prob, world=1, num_sms=148, max_aggregates=74):
    """Plan of the row-distributed two-level PCG on the CPU (rows over world x G virtual CTAs, rank-aligned aggregates, halo masks);
    the library verifies its invariants and raises CubaError if one fails."""
    L = load_library()
    P, keep = _problem_struct(prob)
    info = np.zeros(len(PCG5_PLAN_FIELDS), np.int32)
    _check(L.cuba_debug_pcg5_plan(C.byref(P), int(world), int(num_sms), int(max_aggregates), _p(info)))
    return dict(zip(PCG5_PLAN_FIELDS, (int(v) for v in info)))


def pcg5_plan_apc_host(prob, aggs_per_cta, world=1, num_sms=132, max_aggregates=148):
    """pcg5_plan_host with `aggs_per_cta` aggregates per CTA (the one-GPU tuned kernel's coarse space); also returns "hash", an
    FNV-1a hash over every array of the plan"""
    L = load_library()
    P, keep = _problem_struct(prob)
    info = np.zeros(len(PCG5_PLAN_FIELDS), np.int32)
    h = C.c_uint64(0)
    _check(L.cuba_debug_pcg5_plan_apc(C.byref(P), int(world), int(num_sms), int(max_aggregates), int(aggs_per_cta), _p(info), C.byref(h)))
    out = dict(zip(PCG5_PLAN_FIELDS, (int(v) for v in info)))
    out["hash"] = int(h.value)
    return out


LINEAR_SOLVERS = {"pcg": 0, "dense": 1}            # include/cuba_b200.h: CUBA_SOLVER_PCG, CUBA_SOLVER_DENSE_CHOLESKY
DENSE_MAX_POSES = 2730                             # the direct solver's cap on free poses (n = 6 numP <= 16380)
DENSE_LAYOUT_FIELDS = ("numP", "n", "nt", "tiles", "tile_mb")


def set_linear_solver_raw(value):
    """cuba_engine_set_linear_solver on no engine: the library checks the value before the engine, so this reaches no device; for
    tests of that order"""
    rc = load_library().cuba_engine_set_linear_solver(None, int(value))
    return rc, load_library().cuba_last_error().decode()


def dense_layout_host(prob):
    """The direct solver's layout for the problem on the CPU (include/cuba_b200.h: cuba_debug_dense_layout): dict of
    DENSE_LAYOUT_FIELDS and "map", the full-BSR block behind every block (i >= j) of the packed lower block triangle (-1: none)"""
    L = load_library()
    P, keep = _problem_struct(prob)
    info = np.zeros(len(DENSE_LAYOUT_FIELDS), np.int32)
    m = np.zeros(prob.numP * (prob.numP + 1) // 2, np.int32)
    _check(L.cuba_debug_dense_layout(C.byref(P), _p(info), _p(m)))
    out = dict(zip(DENSE_LAYOUT_FIELDS, (int(v) for v in info)))
    out["map"] = m
    return out


# cuba_debug_pcg5_ranks: plan[] fields
PCG5_RANKS_PLAN_FIELDS = ("G", "gs", "A", "needMax", "maxRows", "halo", "big", "cinfo")
PCG5T_LAYOUT_FIELDS = ("ok", "aggs_per_cta", "capBlocks", "streamed_blocks", "zhInSmem", "total_bytes", "blk_bytes", "rsu_bytes",
                       "staging_bytes", "rc_bytes", "zh_bytes", "slice_bytes")
H100_SMEM_BUDGET = 227 * 1024 - 2048     # what set_problem leaves to k_pcg5t's dynamic shared memory on an H100


def pcg5t_layout_host(prob, aggs_per_cta_top=2, num_sms=132, scalar_bytes=8, smem_budget=H100_SMEM_BUDGET):
    """Shared-memory layout of the one-GPU tuned PCG kernel as set_problem would pick it (the largest number of aggregates per CTA
    <= aggs_per_cta_top whose plan fits smem_budget bytes), on the CPU"""
    L = load_library()
    P, keep = _problem_struct(prob)
    info = np.zeros(len(PCG5T_LAYOUT_FIELDS), np.int32)
    _check(L.cuba_debug_pcg5t_layout(C.byref(P), int(num_sms), int(aggs_per_cta_top), int(scalar_bytes), int(smem_budget), _p(info)))
    return dict(zip(PCG5T_LAYOUT_FIELDS, (int(v) for v in info)))


class Engine:
    """One optimizer instance on one GPU (reference: one CudaBundleAdjustment per thread/device).

    The kernel-selecting options take only the values that name a kernel (cuba_config.reserved[] in include/cuba_b200.h);
    any other makes the constructor raise CubaError before a device is touched:
      pcg_variant    0 automatic (default), 7 / 8 automatic with the rows never / always distributed over the ranks,
                     2 k_pcg2, 3 k_pcg4, 4 k_pcg3, 5 two-level k_pcg5, 6 block-Jacobi k_pcg5
      jh_variant     0 k_linearize_landmark4 (default), 7 / 8 / 9 its three-stage / 5 / 6 CTAs-per-SM shapes,
                     1..4 the first-generation kernel's tile shapes
      schur_variant  0 / 3 k_schur3 (default), 5 landmark tiles on the fp64 tensor pipe (k_schur3 where that cannot run)
    """

    def __init__(self, device=-1, use_fp32=False, pcg_max_iters=0, pcg_tol=0.0, pcg_variant=0, structure_on_host=False, jh_variant=0, schur_variant=0,
                 coarse_refresh=0, two_level_switch=0, max_aggregates=0):
        self.L = load_library()
        res = (C.c_int * 7)()
        res[0] = int(pcg_variant)
        res[1] = int(bool(structure_on_host))
        res[2] = int(jh_variant)
        res[3] = int(schur_variant)
        res[4] = int(coarse_refresh)
        res[5] = int(two_level_switch)
        res[6] = int(max_aggregates)
        cfg = _Config(device, 2 if use_fp32 == "mixed" else int(use_fp32), int(pcg_max_iters), float(pcg_tol), 1, res)
        h = C.c_void_p()
        _check(self.L.cuba_engine_create(C.byref(cfg), C.byref(h)))
        self.h = h
        d = C.c_int(-1)
        _check(self.L.cuba_engine_get_device(h, C.byref(d)))
        self._device = d.value          # the device the engine runs on, device=-1 resolved
        self.sizes = None
        self._stats = []

    def close(self):
        if getattr(self, "h", None):
            self.L.cuba_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- reference API mirror ------------------------------------------------------------------------
    def set_robust_kernels(self, kernel_type, delta, edge_type):
        """setRobustKernels(kernelType, delta, edgeType), include/cuda_bundle_adjustment.h:93"""
        _check(self.L.cuba_engine_set_robust_kernel(self.h, int(edge_type), int(kernel_type), float(delta)))

    def set_comm(self, rank, world, unique_id=None):
        buf = None if unique_id is None else (C.c_char * 128).from_buffer_copy(bytes(unique_id))
        _check(self.L.cuba_engine_set_comm(self.h, rank, world, buf))

    @staticmethod
    def comm_unique_id():
        buf = (C.c_char * 128)()
        _check(load_library().cuba_comm_unique_id(buf))
        return bytes(buf)

    def initialize(self, prob):
        """initialize() + buildStructure(): upload the flat problem, build all index structures."""
        P, keep = _problem_struct(prob)
        _check(self.L.cuba_engine_set_problem(self.h, C.byref(P)))
        sz = _Sizes()
        _check(self.L.cuba_engine_get_sizes(self.h, C.byref(sz)))
        self.sizes = {n: getattr(sz, n) for n, _ in _Sizes._fields_}
        self._stats = []
        return self.sizes

    def set_linear_solver(self, solver):
        """"pcg" (default: the PCG family of pcg_variant) or "dense" (dense fp64 Cholesky of S, at most DENSE_MAX_POSES free poses);
        applies from the next initialize()"""
        if solver not in LINEAR_SOLVERS:
            raise ValueError("linear solver %r: one of %s" % (solver, ", ".join(LINEAR_SOLVERS)))
        _check(self.L.cuba_engine_set_linear_solver(self.h, LINEAR_SOLVERS[solver]))

    def set_structure_reuse(self, enable):
        _check(self.L.cuba_engine_set_structure_reuse(self.h, int(bool(enable))))

    def structure_reuses(self):
        n = C.c_longlong(0)
        _check(self.L.cuba_engine_get_structure_reuses(self.h, C.byref(n)))
        return n.value

    def set_state(self, q, t, Xw):
        q, t, Xw = (np.ascontiguousarray(a, dtype=np.float64) for a in (q, t, Xw))
        _check(self.L.cuba_engine_set_state(self.h, _p(q), _p(t), _p(Xw)))

    def reset_state(self):
        _check(self.L.cuba_engine_reset_state(self.h))

    def stream_ptr(self):
        s = C.c_void_p()
        _check(self.L.cuba_engine_get_stream(self.h, C.byref(s)))
        return s.value or 0

    def flush_l2(self):
        _check(self.L.cuba_engine_flush_l2(self.h))

    def optimize(self, niterations):
        stats = (_IterStat * max(niterations, 1))()
        n = C.c_int(0)
        _check(self.L.cuba_engine_optimize(self.h, niterations, stats, C.byref(n)))
        self._stats = [dict(iteration=s.iteration, trials=s.trials, chi2=s.chi2, lambda_=s.lambda_, pcg_iters=s.pcg_iters,
                            pcg_failed=s.pcg_failed) for s in stats[:n.value]]
        return self._stats

    def batch_statistics(self):
        return [(s["iteration"], s["chi2"]) for s in self._stats]

    def time_profile(self):
        sec = np.zeros(len(PROFILE_ITEMS))
        _check(self.L.cuba_engine_get_profile(self.h, _p(sec)))
        return dict(zip(PROFILE_ITEMS, sec.tolist()))

    def state(self):
        s = self.sizes
        q = np.zeros((s["Pall"], 4)); t = np.zeros((s["Pall"], 3)); Xw = np.zeros((s["Lall"], 3))
        _check(self.L.cuba_engine_get_state(self.h, _p(q), _p(t), _p(Xw)))
        return q, t, Xw

    def chi_squared(self):
        out = np.zeros(self.sizes["E2"] + self.sizes["E3"])
        _check(self.L.cuba_engine_get_chi2(self.h, _p(out)))
        return out

    # --- edge levels (g2o Edge::setLevel + initializeOptimization(0)) ------------------------------------
    def set_edge_levels(self, levels):
        """levels[E2+E3] in edge-id order, 0 = optimised, non-zero = left out of the objective and the normal equations; None = all 0"""
        if levels is None:
            _check(self.L.cuba_engine_set_edge_levels(self.h, None))
            return
        lv = np.ascontiguousarray(np.asarray(levels) != 0, dtype=np.uint8)
        assert lv.shape == (self.sizes["E2"] + self.sizes["E3"],), lv.shape
        _check(self.L.cuba_engine_set_edge_levels(self.h, _p(lv)))

    def edge_levels(self):
        out = np.zeros(self.sizes["E2"] + self.sizes["E3"], np.uint8)
        _check(self.L.cuba_engine_get_edge_levels(self.h, _p(out)))
        return out

    def classify_edges(self, chi2_mono, chi2_stereo, depth=True, reinclude=False):
        """ORB-SLAM2's outlier test on the device at the current estimate (include/cuba_b200.h: cuba_engine_classify_edges)"""
        counts = np.zeros(4, np.int32)
        flags = (1 if depth else 0) | (2 if reinclude else 0)
        _check(self.L.cuba_engine_classify_edges(self.h, float(chi2_mono), float(chi2_stereo), flags, _p(counts)))
        return dict(zip(("included_mono", "included_stereo", "excluded", "reincluded"), (int(v) for v in counts)))

    # --- batched pose optimisation (ORB-SLAM2's PoseOptimization over many frames in one launch) ------------------------------------
    @staticmethod
    def _rounds_struct(rounds):
        rs = (_PoseRound * max(len(rounds), 1))()
        for k, r in enumerate(rounds):
            rs[k].iterations = int(r.iterations)
            rs[k].kernel_type[0], rs[k].kernel_type[1] = int(r.kernel[0]), int(r.kernel[1])
            rs[k].delta[0], rs[k].delta[1] = float(r.delta[0]), float(r.delta[1])
            rs[k].restart = int(bool(r.restart))
            rs[k].chi2_mono, rs[k].chi2_stereo = float(r.chi2_mono), float(r.chi2_stereo)
            rs[k].flags = (1 if r.depth else 0) | (2 if r.reinclude else 0)
        return rs

    @staticmethod
    def _round_stats(stats, nstats, rounds):
        """one problem's structured stats [sum of iterations] and nstats [R] as, per round, the list optimize() returns"""
        off = np.concatenate([[0], np.cumsum([int(x.iterations) for x in rounds])])
        return [[dict(iteration=int(s["iteration"]), trials=int(s["trials"]), chi2=float(s["chi2"]), lambda_=float(s["lambda_"]),
                      pcg_iters=int(s["pcg_iters"]), pcg_failed=int(s["pcg_failed"])) for s in stats[off[k]:off[k] + nstats[k]]]
                for k in range(len(rounds))]

    def optimize_poses_flat(self, q, t, cam, ptr2, X2, meas2, omega2, ptr3, X3, meas3, omega3, rounds, B=None, E2=None, E3=None):
        """cuba_engine_optimize_poses on flat arrays (include/cuba_b200.h); B / E2 / E3 default to the array sizes.  Returns a dict of
        q [B,4], t [B,3], levels [E2+E3] (mono then stereo), counts [B,R,4], stats [B,sum of iterations] (structured) and nstats [B,R]."""
        q, t, cam = _f64(q, 4), _f64(t, 3), _f64(cam, 5)
        X2, meas2, omega2, X3, meas3, omega3 = _f64(X2, 3), _f64(meas2, 2), _f64(omega2, 1), _f64(X3, 3), _f64(meas3, 3), _f64(omega3, 1)
        ptr2 = np.ascontiguousarray(ptr2, dtype=np.int32); ptr3 = np.ascontiguousarray(ptr3, dtype=np.int32)
        B = len(q) if B is None else int(B)
        E2 = len(omega2) if E2 is None else int(E2)
        E3 = len(omega3) if E3 is None else int(E3)
        nb, R = max(B, 0), len(rounds)
        S = sum(max(int(r.iterations), 0) for r in rounds)
        out = dict(q=np.zeros((nb, 4)), t=np.zeros((nb, 3)), levels=np.zeros(max(E2, 0) + max(E3, 0), np.uint8),
                   counts=np.zeros((nb, R, 4), np.int32), stats=(_IterStat * max(nb * S, 1))(), nstats=np.zeros((nb, R), np.int32))
        batch = _PoseBatch(B, E2, E3, _p(q), _p(t), _p(cam), _p(ptr2), _p(X2), _p(meas2), _p(omega2), _p(ptr3), _p(X3), _p(meas3), _p(omega3))
        _check(self.L.cuba_engine_optimize_poses(self.h, C.byref(batch), R, self._rounds_struct(rounds), _p(out["q"]), _p(out["t"]),
                                                 _p(out["levels"]), _p(out["counts"]), out["stats"], _p(out["nstats"])))
        out["stats"] = np.frombuffer(out["stats"], dtype=ITER_STAT_DTYPE)[:nb * S].reshape(nb, S).copy()
        return out

    def optimize_poses(self, frames, rounds):
        """Refines every frame's pose against its fixed points under the round schedule (list of PoseRound) in one launch.  frames:
        graphio.PoseFrame objects.  Returns, per frame, a dict of q [4], t [3], levels (the frame's mono edges then its stereo edges),
        counts [R,4] (included mono, included stereo, newly excluded, re-included after each round) and stats (per round, the
        iteration statistics as optimize() returns them)."""
        a = graphio.pose_batch_arrays(frames)
        ptr2, ptr3 = a["ptr2"], a["ptr3"]
        r = self.optimize_poses_flat(rounds=rounds, **a)
        E2 = int(ptr2[-1])
        return [dict(q=r["q"][b], t=r["t"][b], counts=r["counts"][b], stats=self._round_stats(r["stats"][b], r["nstats"][b], rounds),
                     levels=np.concatenate([r["levels"][ptr2[b]:ptr2[b + 1]], r["levels"][E2 + ptr3[b]:E2 + ptr3[b + 1]]]))
                for b in range(len(frames))]

    # --- batched structure-only refinement (many map points against fixed poses in one launch) ----------------------------------------
    def optimize_points_flat(self, Xw, q, t, cam, ptr2, iP2, meas2, omega2, ptr3, iP3, meas3, omega3, rounds, B=None, P=None, E2=None,
                             E3=None):
        """cuba_engine_optimize_points on flat arrays (include/cuba_b200.h); B / P / E2 / E3 default to the array sizes.  Returns a dict
        of Xw [B,3], levels [E2+E3] (mono then stereo), counts [B,R,4], stats [B,sum of iterations] (structured) and nstats [B,R]."""
        i32 = lambda a: np.ascontiguousarray(np.asarray(a).reshape(-1), dtype=np.int32)
        Xw, q, t, cam = _f64(Xw, 3), _f64(q, 4), _f64(t, 3), _f64(cam, 5)
        meas2, omega2, meas3, omega3 = _f64(meas2, 2), _f64(omega2, 1), _f64(meas3, 3), _f64(omega3, 1)
        ptr2, iP2, ptr3, iP3 = i32(ptr2), i32(iP2), i32(ptr3), i32(iP3)
        B = len(Xw) if B is None else int(B)
        P = len(q) if P is None else int(P)
        E2 = len(omega2) if E2 is None else int(E2)
        E3 = len(omega3) if E3 is None else int(E3)
        nb, R = max(B, 0), len(rounds)
        S = sum(max(int(r.iterations), 0) for r in rounds)
        out = dict(Xw=np.zeros((nb, 3)), levels=np.zeros(max(E2, 0) + max(E3, 0), np.uint8), counts=np.zeros((nb, R, 4), np.int32),
                   stats=(_IterStat * max(nb * S, 1))(), nstats=np.zeros((nb, R), np.int32))
        batch = _PointBatch(B, P, E2, E3, _p(Xw), _p(q), _p(t), _p(cam), _p(ptr2), _p(iP2), _p(meas2), _p(omega2), _p(ptr3), _p(iP3),
                            _p(meas3), _p(omega3))
        _check(self.L.cuba_engine_optimize_points(self.h, C.byref(batch), R, self._rounds_struct(rounds), _p(out["Xw"]), _p(out["levels"]),
                                                  _p(out["counts"]), out["stats"], _p(out["nstats"])))
        out["stats"] = np.frombuffer(out["stats"], dtype=ITER_STAT_DTYPE)[:nb * S].reshape(nb, S).copy()
        return out

    def optimize_points(self, batch, rounds):
        """Refines every point of a graphio.PointBatch against its fixed poses under the round schedule (list of PoseRound; restart =
        from the point's input position) in one launch.  Returns, per point, a dict of Xw [3], levels (the point's mono edges then its
        stereo edges), counts [R,4] (included mono, included stereo, newly excluded, re-included after each round) and stats (per round,
        the iteration statistics as optimize() returns them)."""
        r = self.optimize_points_flat(rounds=rounds, **batch.arrays())
        ptr2, ptr3, E2 = batch.ptr2, batch.ptr3, int(batch.ptr2[-1])
        return [dict(Xw=r["Xw"][b], counts=r["counts"][b], stats=self._round_stats(r["stats"][b], r["nstats"][b], rounds),
                     levels=np.concatenate([r["levels"][ptr2[b]:ptr2[b + 1]], r["levels"][E2 + ptr3[b]:E2 + ptr3[b + 1]]]))
                for b in range(batch.B)]

    # --- structure-only refinement of the held problem's landmarks in place (include/cuba_b200.h: cuba_engine_optimize_landmarks) ------
    def _landmark_count(self, what, landmarks):
        if self.sizes is None:
            raise CubaError("%s before initialize / initialize_device" % what)
        return self.sizes["numL"] if landmarks is None else int(landmarks.shape[0]) if landmarks.ndim == 1 else -1

    def optimize_landmarks(self, rounds, landmarks=None, with_stats=False):
        """Refines the listed free landmarks of the held problem (int array of iL in [0, numL), no repeats; None = every free landmark)
        against the current poses, in place, under the round schedule (list of PoseRound; restart = from the landmark's position on
        entry), starting from the edges' current levels.  Returns a dict of counts [R,4] (included mono, included stereo, newly
        excluded, re-included over the refined landmarks' edges after each round), nstats [n,R] and, with with_stats, stats [n, sum of
        iterations] (the structured array of the _flat methods)."""
        what = "optimize_landmarks"
        lst = None if landmarks is None else np.ascontiguousarray(np.asarray(landmarks).reshape(-1), dtype=np.int32)
        n = self._landmark_count(what, lst)
        R = len(rounds)
        S = sum(max(int(r.iterations), 0) for r in rounds)
        out = dict(counts=np.zeros((R, 4), np.int32), nstats=np.zeros((n, R), np.int32))
        st = (_IterStat * max(n * S, 1))() if with_stats else None
        _check(self.L.cuba_engine_optimize_landmarks(self.h, _p(lst), n, R, self._rounds_struct(rounds), _p(out["counts"]), st,
                                                     _p(out["nstats"])))
        if with_stats:
            out["stats"] = np.frombuffer(st, dtype=ITER_STAT_DTYPE)[:n * S].reshape(n, S).copy()
        return out

    def optimize_landmarks_device(self, rounds, landmarks=None, with_stats=True, out=None):
        """optimize_landmarks with the list (an int32 CUDA tensor [n] of the engine's device, or None) and the per-landmark outputs in
        device memory, on torch.cuda.current_stream(); one host read-back of the counts.  Returns a dict of counts (numpy [R,4]),
        nstats (int32 CUDA [n,R]) and stats (float64 CUDA [n, sum of iterations, 4] words holding cuba_iter_stat, for stats_view(); None
        without with_stats).  out: an earlier result dict to write nstats / stats into; it must fit exactly.  A list entry outside [0,
        numL) or repeated raises CubaError, with the engine and the outputs unchanged."""
        what = "optimize_landmarks_device"
        import torch
        self._check_tensors(what, [("landmarks", landmarks, torch.int32, None)])
        if landmarks is not None and landmarks.dim() != 1:
            raise ValueError("%s: landmarks must be one-dimensional, got shape %s" % (what, tuple(landmarks.shape)))
        n = self._landmark_count(what, landmarks)
        R = len(rounds)
        S = sum(max(int(r.iterations), 0) for r in rounds)
        spec = dict(nstats=((n, R), torch.int32), stats=((n, S, 4), torch.float64))
        out, _, torch = self._device_call(what, [("landmarks", landmarks)], spec, with_stats, out, None)
        counts = np.zeros((R, 4), np.int32)
        _check(self.L.cuba_engine_optimize_landmarks_device(self.h, _dp(landmarks), n, R, self._rounds_struct(rounds), _p(counts),
                                                            _dp(out.get("stats")), _dp(out["nstats"]), C.c_void_p(self._torch_stream())))
        return dict(counts=counts, nstats=out["nstats"], stats=out.get("stats"))

    # --- batched Sim(3) alignment (ORB-SLAM2's OptimizeSim3 over many keyframe pairs in one launch) ------------------------------------
    def optimize_sim3_flat(self, ptr, q, t, s, cam1, cam2, fix_scale, X1, X2, obs1, obs2, omega1, omega2, params=None, B=None, N=None):
        """cuba_engine_optimize_sim3 on flat arrays (include/cuba_b200.h); fix_scale may be None; B / N default to the array sizes.
        Returns a dict of q [B,4], t [B,3], s [B], levels [N], ninliers [B], stats [B, iterations + max(bad, good)] (structured) and
        nstats [B,2]."""
        params = Sim3Params() if params is None else params
        q, t, s, cam1, cam2 = _f64(q, 4), _f64(t, 3), _f64(s, 1), _f64(cam1, 4), _f64(cam2, 4)
        X1, X2, obs1, obs2, omega1, omega2 = _f64(X1, 3), _f64(X2, 3), _f64(obs1, 2), _f64(obs2, 2), _f64(omega1, 1), _f64(omega2, 1)
        ptr = np.ascontiguousarray(ptr, dtype=np.int32)
        fix = None if fix_scale is None else np.ascontiguousarray(fix_scale, dtype=np.int32)
        B = len(s) if B is None else int(B)
        N = len(omega1) if N is None else int(N)
        nb = max(B, 0)
        S = max(int(params.iterations), 0) + max(int(params.iterations_bad), int(params.iterations_good), 0)
        out = dict(q=np.zeros((nb, 4)), t=np.zeros((nb, 3)), s=np.zeros(nb), levels=np.zeros(max(N, 0), np.uint8),
                   ninliers=np.zeros(nb, np.int32), stats=(_IterStat * max(nb * S, 1))(), nstats=np.zeros((nb, 2), np.int32))
        batch = _Sim3Batch(B, N, _p(ptr), _p(q), _p(t), _p(s), _p(cam1), _p(cam2), _p(fix), _p(X1), _p(X2), _p(obs1), _p(obs2),
                           _p(omega1), _p(omega2))
        prm = _Sim3Params(float(params.chi2), int(params.iterations), int(params.iterations_bad), int(params.iterations_good),
                          int(params.min_pairs))
        _check(self.L.cuba_engine_optimize_sim3(self.h, C.byref(batch), C.byref(prm), _p(out["q"]), _p(out["t"]), _p(out["s"]),
                                                _p(out["levels"]), _p(out["ninliers"]), out["stats"], _p(out["nstats"])))
        out["stats"] = np.frombuffer(out["stats"], dtype=ITER_STAT_DTYPE)[:nb * S].reshape(nb, S).copy()
        return out

    def optimize_sim3(self, problems, params=None):
        """Refines S12 of every problem (graphio.Sim3Problem) under OptimizeSim3's schedule (Sim3Params) in one launch.  Returns, per
        problem, a dict of q [4], t [3], s, levels (0/1 per pair), ninliers and stats (the iteration statistics of the first and of
        the second optimize, as optimize() returns them)."""
        params = Sim3Params() if params is None else params
        a = graphio.sim3_batch_arrays(problems)
        ptr = a["ptr"]
        r = self.optimize_sim3_flat(params=params, **a)
        off = (0, int(params.iterations))
        res = []
        for b in range(len(problems)):
            stats = []
            for k in range(2):
                rows = r["stats"][b, off[k]:off[k] + r["nstats"][b, k]]
                stats.append([dict(iteration=int(x["iteration"]), trials=int(x["trials"]), chi2=float(x["chi2"]), lambda_=float(x["lambda_"]),
                                   pcg_iters=int(x["pcg_iters"]), pcg_failed=int(x["pcg_failed"])) for x in rows])
            res.append(dict(q=r["q"][b], t=r["t"][b], s=float(r["s"][b]), levels=r["levels"][ptr[b]:ptr[b + 1]].copy(),
                            ninliers=int(r["ninliers"][b]), stats=stats))
        return res

    # --- the two batches on device-resident data (include/cuba_b200.h: cuba_engine_optimize_*_device) --------------------------------
    # Every tensor whose address reaches the library -- inputs, outputs (fresh or reused through out=) and the workspace -- is checked
    # here first: the library cannot see the size or the device of a device buffer.
    @staticmethod
    def _check_tensors(what, arrays):
        """arrays: (name, tensor or None, torch dtype, shape or None).  Type, dtype, contiguity and, where given, shape."""
        import torch
        for name, a, dt, shape in arrays:
            if a is None:
                continue
            if not isinstance(a, torch.Tensor):
                raise TypeError("%s: %s must be a torch tensor, got %s" % (what, name, type(a).__name__))
            if a.dtype != dt:
                raise TypeError("%s: %s is %s, must be %s" % (what, name, a.dtype, dt))
            if not a.is_contiguous():
                raise ValueError("%s: %s is not contiguous" % (what, name))
            if shape is not None and tuple(a.shape) != tuple(shape):
                raise ValueError("%s: %s has shape %s, must be %s" % (what, name, tuple(a.shape), tuple(shape)))

    def _check_devices(self, what, arrays):
        for name, a in arrays:
            if a is not None and (a.device.type != "cuda" or a.device.index != self._device):
                raise ValueError("%s: %s is on %s, the engine on cuda:%d" % (what, name, a.device, self._device))

    @staticmethod
    def _count(what, name, a, width, n=None):
        """a.numel() / width, checked against n when given"""
        k = a.numel() // width
        if a.numel() != k * width or (n is not None and k != n):
            raise ValueError("%s: %s has %d elements, expected %s x %d" % (what, name, a.numel(), "a multiple" if n is None else n, width))
        return k

    def _device_call(self, what, inputs, out_spec, with_stats, out, workspace):
        """the host-side checks and allocations of a device call.  inputs: (name, tensor) already checked for dtype and shape;
        out_spec: {name: (shape, dtype)} of every output.  A reused `out` must hold exactly those tensors (stats absent or None
        without with_stats); a reused workspace must be a float64 CUDA tensor (the library checks its size).  Returns (out,
        workspace or None, torch)."""
        import torch
        if out is not None:
            if not isinstance(out, dict):
                raise TypeError("%s: out must be the dict an earlier call returned" % what)
            if (out.get("stats") is not None) != bool(with_stats):
                raise ValueError("%s: out%s stats, with_stats is %s" % (what, " has" if out.get("stats") is not None else " has no", with_stats))
            missing = [k for k in out_spec if k != "stats" and k not in out]
            if missing:
                raise ValueError("%s: out lacks %s" % (what, ", ".join(missing)))
            self._check_tensors(what, [("out[%r]" % k, out.get(k), dt, shape) for k, (shape, dt) in out_spec.items()])
        self._check_tensors(what, [("workspace", workspace, torch.float64, None)])
        if workspace is not None and workspace.dim() != 1:
            raise ValueError("%s: workspace must be one-dimensional" % what)
        self._check_devices(what, [("workspace", workspace)] + ([("out[%r]" % k, out.get(k)) for k in out_spec] if out is not None else []) +
                            list(inputs))
        if out is None:
            dev = torch.device("cuda", self._device)
            out = {k: None if (k == "stats" and not with_stats) else torch.empty(shape, dtype=dt, device=dev) for k, (shape, dt) in out_spec.items()}
        return out, workspace, torch

    def _workspace(self, torch, workspace, need):
        return torch.empty((need + 7) // 8, dtype=torch.float64, device=torch.device("cuda", self._device)) if workspace is None else workspace

    def _torch_stream(self):
        """torch.cuda.current_stream() of the engine's device as the C ABI takes it"""
        import torch
        h = torch.cuda.current_stream(self._device).cuda_stream
        return h if h else 1          # handle 0 is the legacy default stream: cudaStreamLegacy, not "the engine's stream"

    def optimize_poses_device(self, q, t, cam, ptr2, X2, meas2, omega2, ptr3, X3, meas3, omega3, rounds, with_stats=True, out=None,
                              workspace=None):
        """cuba_engine_optimize_poses_device: optimize_poses_flat on torch CUDA tensors of the engine's device (float64, ptr2 / ptr3
        int32, all contiguous), on torch.cuda.current_stream(); no host synchronisation, no host<->device copy.  Returns a dict of CUDA
        tensors with optimize_poses_flat's keys and shapes, except stats: [B, sum of iterations, 4] float64 words holding
        cuba_iter_stat, which stats_view() turns into the structured array; plus "status" (int32 [1], 0 = ok, else the bits of
        BATCH_STATUS; no output is written then) and "workspace".  out / workspace: an earlier result dict and its "workspace" entry,
        to run again into the same tensors (a CUDA graph replays into them); they must fit this batch exactly."""
        what = "optimize_poses_device"
        import torch
        f64, i32 = torch.float64, torch.int32
        inputs = [("q", q, f64), ("t", t, f64), ("cam", cam, f64), ("ptr2", ptr2, i32), ("X2", X2, f64), ("meas2", meas2, f64),
                  ("omega2", omega2, f64), ("ptr3", ptr3, i32), ("X3", X3, f64), ("meas3", meas3, f64), ("omega3", omega3, f64)]
        self._check_tensors(what, [(n, a, dt, None) for n, a, dt in inputs])
        B = self._count(what, "q", q, 4)
        for name, a, w in (("t", t, 3), ("cam", cam, 5)):
            self._count(what, name, a, w, B)
        for name, a in (("ptr2", ptr2), ("ptr3", ptr3)):
            self._count(what, name, a, 1, B + 1)
        E2, E3 = omega2.numel(), omega3.numel()
        for name, a, w, n in (("X2", X2, 3, E2), ("meas2", meas2, 2, E2), ("X3", X3, 3, E3), ("meas3", meas3, 3, E3)):
            self._count(what, name, a, w, n)
        R = len(rounds)
        S = sum(max(int(r.iterations), 0) for r in rounds)
        spec = dict(q=((B, 4), f64), t=((B, 3), f64), levels=((E2 + E3,), torch.uint8), counts=((B, R, 4), i32), stats=((B, S, 4), f64),
                    nstats=((B, R), i32), status=((1,), i32))
        out, workspace, torch = self._device_call(what, [(n, a) for n, a, _ in inputs], spec, with_stats, out, workspace)
        rs = self._rounds_struct(rounds)
        workspace = self._workspace(torch, workspace, int(self.L.cuba_pose_batch_workspace_bytes(B, E2, E3, R, rs, int(bool(with_stats)))))
        batch = _PoseBatch(B, E2, E3, _dp(q), _dp(t), _dp(cam), _dp(ptr2), _dp(X2), _dp(meas2), _dp(omega2), _dp(ptr3), _dp(X3), _dp(meas3),
                           _dp(omega3))
        _check(self.L.cuba_engine_optimize_poses_device(self.h, C.byref(batch), R, rs, _dp(workspace), workspace.numel() * workspace.element_size(),
                                                        _dp(out["q"]), _dp(out["t"]), _dp(out["levels"]), _dp(out["counts"]),
                                                        _dp(out["stats"]), _dp(out["nstats"]), _dp(out["status"]), C.c_void_p(self._torch_stream())))
        out["workspace"] = workspace
        return out

    def optimize_sim3_device(self, ptr, q, t, s, cam1, cam2, fix_scale, X1, X2, obs1, obs2, omega1, omega2, params=None, with_stats=True,
                             out=None, workspace=None):
        """cuba_engine_optimize_sim3_device: optimize_sim3_flat on torch CUDA tensors of the engine's device (float64, ptr and
        fix_scale int32, fix_scale may be None; all contiguous), on torch.cuda.current_stream(); no host synchronisation, no
        host<->device copy.  Returns a dict of CUDA tensors with optimize_sim3_flat's keys and shapes, except stats: [B, iterations +
        max(bad, good), 4] float64 words (stats_view()); plus "status" (int32 [1]; BATCH_STATUS) and "workspace".  out / workspace as
        for optimize_poses_device."""
        what = "optimize_sim3_device"
        params = Sim3Params() if params is None else params
        import torch
        f64, i32 = torch.float64, torch.int32
        inputs = [("ptr", ptr, i32), ("q", q, f64), ("t", t, f64), ("s", s, f64), ("cam1", cam1, f64), ("cam2", cam2, f64),
                  ("fix_scale", fix_scale, i32), ("X1", X1, f64), ("X2", X2, f64), ("obs1", obs1, f64), ("obs2", obs2, f64),
                  ("omega1", omega1, f64), ("omega2", omega2, f64)]
        self._check_tensors(what, [(n, a, dt, None) for n, a, dt in inputs])
        B = s.numel()
        for name, a, w, n in (("q", q, 4, B), ("t", t, 3, B), ("cam1", cam1, 4, B), ("cam2", cam2, 4, B), ("ptr", ptr, 1, B + 1)):
            self._count(what, name, a, w, n)
        if fix_scale is not None:
            self._count(what, "fix_scale", fix_scale, 1, B)
        N = omega1.numel()
        for name, a, w in (("X1", X1, 3), ("X2", X2, 3), ("obs1", obs1, 2), ("obs2", obs2, 2), ("omega2", omega2, 1)):
            self._count(what, name, a, w, N)
        S = max(int(params.iterations), 0) + max(int(params.iterations_bad), int(params.iterations_good), 0)
        spec = dict(q=((B, 4), f64), t=((B, 3), f64), s=((B,), f64), levels=((N,), torch.uint8), ninliers=((B,), i32), stats=((B, S, 4), f64),
                    nstats=((B, 2), i32), status=((1,), i32))
        out, workspace, torch = self._device_call(what, [(n, a) for n, a, _ in inputs], spec, with_stats, out, workspace)
        prm = _Sim3Params(float(params.chi2), int(params.iterations), int(params.iterations_bad), int(params.iterations_good),
                          int(params.min_pairs))
        workspace = self._workspace(torch, workspace, int(self.L.cuba_sim3_batch_workspace_bytes(B, N, C.byref(prm), int(bool(with_stats)))))
        batch = _Sim3Batch(B, N, _dp(ptr), _dp(q), _dp(t), _dp(s), _dp(cam1), _dp(cam2), _dp(fix_scale), _dp(X1), _dp(X2), _dp(obs1), _dp(obs2), _dp(omega1), _dp(omega2))
        _check(self.L.cuba_engine_optimize_sim3_device(self.h, C.byref(batch), C.byref(prm), _dp(workspace),
                                                       workspace.numel() * workspace.element_size(), _dp(out["q"]), _dp(out["t"]), _dp(out["s"]),
                                                       _dp(out["levels"]), _dp(out["ninliers"]), _dp(out["stats"]), _dp(out["nstats"]), _dp(out["status"]),
                                                       C.c_void_p(self._torch_stream())))
        out["workspace"] = workspace
        return out

    def optimize_points_device(self, Xw, q, t, cam, ptr2, iP2, meas2, omega2, ptr3, iP3, meas3, omega3, rounds, with_stats=True, out=None,
                               workspace=None):
        """cuba_engine_optimize_points_device: optimize_points_flat on torch CUDA tensors of the engine's device (float64, ptr2 / ptr3 /
        iP2 / iP3 int32, all contiguous), on torch.cuda.current_stream(); no host synchronisation, no host<->device copy.  Returns a
        dict of CUDA tensors with optimize_points_flat's keys and shapes, except stats: [B, sum of iterations, 4] float64 words
        (stats_view()); plus "status" (int32 [1]; BATCH_STATUS) and "workspace".  out / workspace as for optimize_poses_device."""
        what = "optimize_points_device"
        import torch
        f64, i32 = torch.float64, torch.int32
        inputs = [("Xw", Xw, f64), ("q", q, f64), ("t", t, f64), ("cam", cam, f64), ("ptr2", ptr2, i32), ("iP2", iP2, i32),
                  ("meas2", meas2, f64), ("omega2", omega2, f64), ("ptr3", ptr3, i32), ("iP3", iP3, i32), ("meas3", meas3, f64),
                  ("omega3", omega3, f64)]
        self._check_tensors(what, [(n, a, dt, None) for n, a, dt in inputs])
        B = self._count(what, "Xw", Xw, 3)
        P = self._count(what, "q", q, 4)
        for name, a, w in (("t", t, 3), ("cam", cam, 5)):
            self._count(what, name, a, w, P)
        for name, a in (("ptr2", ptr2), ("ptr3", ptr3)):
            self._count(what, name, a, 1, B + 1)
        E2, E3 = omega2.numel(), omega3.numel()
        for name, a, w, n in (("iP2", iP2, 1, E2), ("meas2", meas2, 2, E2), ("iP3", iP3, 1, E3), ("meas3", meas3, 3, E3)):
            self._count(what, name, a, w, n)
        R = len(rounds)
        S = sum(max(int(r.iterations), 0) for r in rounds)
        spec = dict(Xw=((B, 3), f64), levels=((E2 + E3,), torch.uint8), counts=((B, R, 4), i32), stats=((B, S, 4), f64), nstats=((B, R), i32),
                    status=((1,), i32))
        out, workspace, torch = self._device_call(what, [(n, a) for n, a, _ in inputs], spec, with_stats, out, workspace)
        rs = self._rounds_struct(rounds)
        workspace = self._workspace(torch, workspace, int(self.L.cuba_point_batch_workspace_bytes(B, P, E2, E3, R, rs, int(bool(with_stats)))))
        batch = _PointBatch(B, P, E2, E3, _dp(Xw), _dp(q), _dp(t), _dp(cam), _dp(ptr2), _dp(iP2), _dp(meas2), _dp(omega2), _dp(ptr3), _dp(iP3),
                            _dp(meas3), _dp(omega3))
        _check(self.L.cuba_engine_optimize_points_device(self.h, C.byref(batch), R, rs, _dp(workspace), workspace.numel() * workspace.element_size(),
                                                         _dp(out["Xw"]), _dp(out["levels"]), _dp(out["counts"]), _dp(out["stats"]),
                                                         _dp(out["nstats"]), _dp(out["status"]), C.c_void_p(self._torch_stream())))
        out["workspace"] = workspace
        return out

    # --- the engine's own problem on device-resident data (include/cuba_b200.h: cuba_engine_set_problem_device etc.) ----------------
    # Torch CUDA tensors of the engine's device, checked like the batches' (dtype, contiguity, exact shape, device) before any library
    # call; the work runs on torch.cuda.current_stream(), ordered after what is queued there, and torch's later work after it.
    def _problem_sizes(self, what):
        if self.sizes is None:
            raise CubaError("%s before initialize / initialize_device" % what)
        s = self.sizes
        return s["Pall"], s["Lall"], s["E2"] + s["E3"]

    def _tensors(self, what, arrays):
        """arrays: (name, tensor or None, torch dtype, exact shape)"""
        self._check_tensors(what, arrays)
        self._check_devices(what, [(n, a) for n, a, _, _ in arrays])

    def _empty(self, shape, dtype):
        import torch
        return torch.empty(shape, dtype=dtype, device=torch.device("cuda", self._device))

    def initialize_device(self, prob):
        """initialize() on device-resident arrays: prob is a dict or an object with initialize()'s fields (Pall, numP, Lall, numL and
        q [Pall,4], t [Pall,3], cam [Pall,5], Xw [Lall,3], idx2 [E2,2] int32, meas2 [E2,2], omega2 [E2], idx3 [E3,2] int32, meas3 [E3,3],
        omega3 [E3] as torch CUDA tensors, float64 unless noted; E2 / E3 default to the lengths of omega2 / omega3).  Synchronous like
        initialize(); no bulk host<->device copy.  Returns sizes."""
        what = "initialize_device"
        import torch
        get = (lambda k, d=None: prob.get(k, d)) if isinstance(prob, dict) else (lambda k, d=None: getattr(prob, k, d))
        Pall, numP, Lall, numL = (int(get(k)) for k in ("Pall", "numP", "Lall", "numL"))
        names = ("q", "t", "cam", "Xw", "idx2", "meas2", "omega2", "idx3", "meas3", "omega3")
        a = {n: get(n) for n in names}
        missing = [n for n in names if a[n] is None]
        if missing:
            raise TypeError("%s: prob lacks %s" % (what, ", ".join(missing)))
        f64, i32 = torch.float64, torch.int32
        self._check_tensors(what, [("omega2", a["omega2"], f64, None), ("omega3", a["omega3"], f64, None)])
        E2 = int(get("E2", a["omega2"].shape[0] if a["omega2"].dim() else -1))
        E3 = int(get("E3", a["omega3"].shape[0] if a["omega3"].dim() else -1))
        spec = [("q", f64, (Pall, 4)), ("t", f64, (Pall, 3)), ("cam", f64, (Pall, 5)), ("Xw", f64, (Lall, 3)), ("idx2", i32, (E2, 2)),
                ("meas2", f64, (E2, 2)), ("omega2", f64, (E2,)), ("idx3", i32, (E3, 2)), ("meas3", f64, (E3, 3)), ("omega3", f64, (E3,))]
        self._tensors(what, [(n, a[n], dt, shape) for n, dt, shape in spec])
        p = {n: a[n].data_ptr() for n in a}
        P = _Problem(Pall, numP, Lall, numL, p["q"], p["t"], p["cam"], p["Xw"], E2, p["idx2"], p["meas2"], p["omega2"], E3, p["idx3"],
                     p["meas3"], p["omega3"])
        _check(self.L.cuba_engine_set_problem_device(self.h, C.byref(P), C.c_void_p(self._torch_stream())))
        sz = _Sizes()
        _check(self.L.cuba_engine_get_sizes(self.h, C.byref(sz)))
        self.sizes = {n: getattr(sz, n) for n, _ in _Sizes._fields_}
        self._stats = []
        return self.sizes

    def set_state_device(self, q, t, Xw):
        """set_state() from CUDA tensors q [Pall,4], t [Pall,3], Xw [Lall,3] (float64); no synchronisation"""
        what = "set_state_device"
        import torch
        Pall, Lall, _ = self._problem_sizes(what)
        self._tensors(what, [("q", q, torch.float64, (Pall, 4)), ("t", t, torch.float64, (Pall, 3)), ("Xw", Xw, torch.float64, (Lall, 3))])
        _check(self.L.cuba_engine_set_state_device(self.h, q.data_ptr(), t.data_ptr(), Xw.data_ptr(), C.c_void_p(self._torch_stream())))

    def state_device(self, out=None):
        """state() into CUDA tensors (q [Pall,4], t [Pall,3], Xw [Lall,3], float64), fresh or the tuple `out`; no synchronisation"""
        what = "state_device"
        import torch
        Pall, Lall, _ = self._problem_sizes(what)
        shapes = ((Pall, 4), (Pall, 3), (Lall, 3))
        if out is None:
            out = tuple(self._empty(sh, torch.float64) for sh in shapes)
        elif not isinstance(out, tuple) or len(out) != 3:
            raise TypeError("%s: out must be a tuple (q, t, Xw)" % what)
        self._tensors(what, [(n, a, torch.float64, sh) for n, a, sh in zip(("q", "t", "Xw"), out, shapes)])
        _check(self.L.cuba_engine_get_state_device(self.h, *(a.data_ptr() for a in out), C.c_void_p(self._torch_stream())))
        return out

    def chi_squared_device(self, out=None):
        """chi_squared() into a CUDA tensor [E2+E3] float64 (fresh or `out`); no synchronisation"""
        what = "chi_squared_device"
        import torch
        _, _, E = self._problem_sizes(what)
        out = self._empty((E,), torch.float64) if out is None else out
        self._tensors(what, [("out", out, torch.float64, (E,))])
        _check(self.L.cuba_engine_get_chi2_device(self.h, out.data_ptr(), C.c_void_p(self._torch_stream())))
        return out

    def set_edge_levels_device(self, levels):
        """set_edge_levels() from a CUDA tensor [E2+E3] uint8 (0 = optimised, non-zero = left out), or None = all 0; waits for one
        8-byte count"""
        what = "set_edge_levels_device"
        import torch
        _, _, E = self._problem_sizes(what)
        self._tensors(what, [("levels", levels, torch.uint8, (E,))])
        _check(self.L.cuba_engine_set_edge_levels_device(self.h, None if levels is None else levels.data_ptr(), C.c_void_p(self._torch_stream())))

    def edge_levels_device(self, out=None):
        """edge_levels() into a CUDA tensor [E2+E3] uint8 (fresh or `out`); no synchronisation"""
        what = "edge_levels_device"
        import torch
        _, _, E = self._problem_sizes(what)
        out = self._empty((E,), torch.uint8) if out is None else out
        self._tensors(what, [("out", out, torch.uint8, (E,))])
        _check(self.L.cuba_engine_get_edge_levels_device(self.h, out.data_ptr(), C.c_void_p(self._torch_stream())))
        return out

    def launch_count(self):
        n = C.c_longlong(0)
        _check(self.L.cuba_engine_get_launch_count(self.h, C.byref(n)))
        return n.value

    # --- stages ----------------------------------------------------------------------------------------
    def linearize(self):
        v = C.c_double(0)
        _check(self.L.cuba_stage_linearize(self.h, C.byref(v)))
        return v.value

    def max_diagonal(self):
        v = C.c_double(0)
        _check(self.L.cuba_stage_max_diagonal(self.h, C.byref(v)))
        return v.value

    def solve(self, lam):
        it, ok = C.c_int(0), C.c_int(0)
        _check(self.L.cuba_stage_solve(self.h, float(lam), C.byref(it), C.byref(ok)))
        return it.value, bool(ok.value)

    def update(self, lam):
        chi, sc = C.c_double(0), C.c_double(0)
        _check(self.L.cuba_stage_update(self.h, float(lam), C.byref(chi), C.byref(sc)))
        return chi.value, sc.value

    def commit(self, accept):
        _check(self.L.cuba_stage_commit(self.h, int(bool(accept))))

    def chi2(self):
        v = C.c_double(0)
        _check(self.L.cuba_stage_chi2(self.h, C.byref(v)))
        return v.value

    # --- debug -----------------------------------------------------------------------------------------
    def hpl_structure(self):
        s = self.sizes
        colPtr = np.zeros(s["numL"] + 1, np.int32); rowInd = np.zeros(s["nhpl"], np.int32); e2h = np.zeros(s["E2"] + s["E3"], np.int32)
        _check(self.L.cuba_debug_get_hpl_structure(self.h, _p(colPtr), _p(rowInd), _p(e2h)))
        return colPtr, rowInd, e2h

    def hsc_structure(self):
        s = self.sizes
        rowPtr = np.zeros(s["numP"] + 1, np.int32); colInd = np.zeros(s["nblk"], np.int32)
        _check(self.L.cuba_debug_get_hsc_structure(self.h, _p(rowPtr), _p(colInd)))
        return rowPtr, colInd

    def system(self):
        s = self.sizes
        Hpp = np.zeros((s["numP"], 36)); bp = np.zeros((s["numP"], 6)); Hll = np.zeros((s["numL"], 9)); bl = np.zeros((s["numL"], 3))
        Hpl = np.zeros((s["nhpl"], 18))
        _check(self.L.cuba_debug_get_system(self.h, _p(Hpp), _p(bp), _p(Hll), _p(bl), _p(Hpl)))
        return Hpp, bp, Hll, bl, Hpl

    def schur(self):
        s = self.sizes
        Hsc = np.zeros((s["nblk"], 36)); bsc = np.zeros((s["numP"], 6)); inv = np.zeros((s["numL"], 9))
        _check(self.L.cuba_debug_get_schur(self.h, _p(Hsc), _p(bsc), _p(inv)))
        return Hsc, bsc, inv

    def delta(self):
        s = self.sizes
        xp = np.zeros((s["numP"], 6)); xl = np.zeros((s["numL"], 3))
        _check(self.L.cuba_debug_get_delta(self.h, _p(xp), _p(xl)))
        return xp, xl

    def pcg_info(self):
        """what the last solve ran (include/cuba_b200.h: cuba_debug_get_pcg_info), kernels by name"""
        info = np.zeros(PCG_INFO_LEN, np.int32)
        lam = C.c_double(0)
        _check(self.L.cuba_debug_get_pcg_info(self.h, _p(info), C.byref(lam)))
        out = dict(zip(PCG_INFO_FIELDS, (int(v) for v in info)))
        out["kernel"] = PCG_KERNELS[out["kernel"]]
        out["coarse_kernel"] = COARSE_KERNELS[out["coarse_kernel"]]
        out["two_level"] = bool(out["two_level"])
        out["coarse_lambda"] = lam.value
        return out

    def coarse(self):
        """(aggregate of every free pose, packed lower blocks of Ac = Z^T S Z [A(A+1)/2][36] column-major, fp32 Ac^-1 [6A][6A]) of
        the k_pcg5 coarse level the last two-level solve applied"""
        A = self.pcg_info()["A"]
        agg = np.zeros(self.sizes["numP"], np.int32); AcP = np.zeros((A * (A + 1) // 2, 36)); AcInv = np.zeros((6 * A, 6 * A), np.float32)
        _check(self.L.cuba_debug_get_coarse(self.h, _p(agg), _p(AcP), _p(AcInv)))
        return agg, AcP, AcInv

    def coarse_inverse(self, AcP):
        """(fp32 Ac^-1 [6A][6A], info) of k_coarse_dense run on the packed lower blocks AcP [A(A+1)/2][36] (column-major), as
        coarse() returns them; info 1: not positive definite, Ac^-1 zeroed"""
        AcP = np.ascontiguousarray(AcP, dtype=np.float64)
        nb = AcP.shape[0]
        A = int(round(((8 * nb + 1) ** 0.5 - 1) / 2))
        assert A * (A + 1) // 2 == nb and AcP.shape[1:] == (36,), AcP.shape
        AcInv = np.zeros((6 * A, 6 * A), np.float32)
        info = C.c_int(-1)
        _check(self.L.cuba_debug_coarse_inverse(self.h, _p(AcP), A, _p(AcInv), C.byref(info)))
        return AcInv, info.value

    def debug_dense_solve(self, S, b):
        """(x, info) of the direct solver's kernel on the dense SPD matrix S [n][n] (its lower triangle is read) and b [n], in buffers
        of its own; info 1: not positive definite, x zeroed"""
        S = np.ascontiguousarray(S, dtype=np.float64)
        b = np.ascontiguousarray(b, dtype=np.float64).reshape(-1)
        n = b.size
        assert S.shape == (n, n), (S.shape, n)
        x = np.zeros(n)
        info = C.c_int(-1)
        _check(self.L.cuba_debug_dense_solve(self.h, _p(S), _p(b), n, _p(x), C.byref(info)))
        return x, info.value

    def peer_allreduce(self, parts):
        """the peer all-reduce of a `world`-rank run emulated on this GPU (include/cuba_b200.h: cuba_debug_peer_allreduce): parts
        [calls][world][n], each call's parts loaded in the engine's scalar type; returns every rank's buffer after every call, same shape"""
        parts = np.ascontiguousarray(parts, dtype=np.float64)
        calls, world, n = parts.shape
        out = np.zeros_like(parts)
        _check(self.L.cuba_debug_peer_allreduce(self.h, int(world), int(n), int(calls), _p(parts), _p(out)))
        return out

    def pcg5_ranks(self, world, two_level, nsolves=3):
        """the row-distributed k_pcg5 of a `world`-rank run emulated on this GPU, on the current reduced system (include/cuba_b200.h:
        cuba_debug_pcg5_ranks).  Returns x [nsolves][numP][6], status [nsolves][world] and iters [nsolves][world] of every rank,
        plan (dict of PCG5_RANKS_PLAN_FIELDS), aggRow [A+1] and the fp32 AcInv [6A][6A] (zeros for block-Jacobi)."""
        P = self.sizes["numP"]
        amax = min(P, 148)
        x = np.zeros((nsolves, P, 6)); st = np.zeros((nsolves, world, 2), np.int32); plan = np.zeros(len(PCG5_RANKS_PLAN_FIELDS), np.int32)
        agg = np.zeros(amax + 1, np.int32); AcInv = np.zeros(36 * amax * amax, np.float32)
        _check(self.L.cuba_debug_pcg5_ranks(self.h, int(world), int(bool(two_level)), int(nsolves), _p(x), _p(st), _p(plan), _p(agg), _p(AcInv)))
        pl = dict(zip(PCG5_RANKS_PLAN_FIELDS, (int(v) for v in plan)))
        A = pl["A"]
        return dict(x=x, status=st[:, :, 0].copy(), iters=st[:, :, 1].copy(), plan=pl, aggRow=agg[:A + 1].copy(),
                    AcInv=AcInv[:36 * A * A].reshape(6 * A, 6 * A).copy())

    def bench_stage(self, stage, reps=10, flush_l2=True, lam=1.0):
        ms = C.c_double(0)
        _check(self.L.cuba_bench_stage(self.h, int(stage), int(reps), int(bool(flush_l2)), float(lam), C.byref(ms)))
        return ms.value
