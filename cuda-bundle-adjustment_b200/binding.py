"""ctypes binding of libcuba_b200.so (include/cuba_b200.h).  Mirrors the reference's operator interface
for the hot path: initialize()/optimize(n)/batchStatistics()/timeProfile()/chiSquared()
(reference include/cuda_bundle_adjustment.h:34-125) on a flat problem."""
import ctypes as C
import dataclasses
import os

import numpy as np

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
    "cuba_comm_unique_id", "cuba_engine_set_comm", "cuba_engine_set_problem", "cuba_engine_set_linear_solver", "cuba_engine_set_structure_reuse", "cuba_engine_get_structure_reuses", "cuba_engine_set_state", "cuba_engine_get_sizes", "cuba_engine_reset_state", "cuba_engine_get_stream", "cuba_engine_flush_l2",
    "cuba_engine_optimize", "cuba_engine_get_state", "cuba_engine_get_chi2", "cuba_engine_set_edge_levels", "cuba_engine_get_edge_levels", "cuba_engine_classify_edges", "cuba_engine_optimize_poses", "cuba_engine_optimize_sim3", "cuba_engine_get_profile",
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
        "cuba_engine_flush_l2": [vp],
        "cuba_engine_optimize": [vp, i, vp, C.POINTER(i)],
        "cuba_engine_get_state": [vp, vp, vp, vp],
        "cuba_engine_get_chi2": [vp, vp],
        "cuba_engine_set_edge_levels": [vp, vp],
        "cuba_engine_get_edge_levels": [vp, vp],
        "cuba_engine_classify_edges": [vp, d, d, i, vp],
        "cuba_engine_optimize_poses": [vp, C.POINTER(_PoseBatch), i, vp, vp, vp, vp, vp, vp, vp],
        "cuba_engine_optimize_sim3": [vp, C.POINTER(_Sim3Batch), C.POINTER(_Sim3Params), vp, vp, vp, vp, vp, vp, vp],
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
    _lib = L
    return L


def _check(rc):
    if rc != 0:
        raise CubaError("cuba error %d: %s" % (rc, load_library().cuba_last_error().decode()))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


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

    def optimize_poses_flat(self, q, t, cam, ptr2, X2, meas2, omega2, ptr3, X3, meas3, omega3, rounds, B=None, E2=None, E3=None):
        """cuba_engine_optimize_poses on flat arrays (include/cuba_b200.h); B / E2 / E3 default to the array sizes.  Returns a dict of
        q [B,4], t [B,3], levels [E2+E3] (mono then stereo), counts [B,R,4], stats [B,sum of iterations] (structured) and nstats [B,R]."""
        f64 = lambda a, w: np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1, w) if w > 1 else np.asarray(a, dtype=np.float64).reshape(-1))
        q, t, cam = f64(q, 4), f64(t, 3), f64(cam, 5)
        X2, meas2, omega2, X3, meas3, omega3 = f64(X2, 3), f64(meas2, 2), f64(omega2, 1), f64(X3, 3), f64(meas3, 3), f64(omega3, 1)
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
        st = np.frombuffer(out["stats"], dtype=np.dtype([("iteration", "<i4"), ("trials", "<i4"), ("chi2", "<f8"), ("lambda_", "<f8"),
                                                          ("pcg_iters", "<i4"), ("pcg_failed", "<i4")]))
        out["stats"] = st[:nb * S].reshape(nb, S).copy()
        return out

    def optimize_poses(self, frames, rounds):
        """Refines every frame's pose against its fixed points under the round schedule (list of PoseRound) in one launch.  frames:
        graphio.PoseFrame objects.  Returns, per frame, a dict of q [4], t [3], levels (the frame's mono edges then its stereo edges),
        counts [R,4] (included mono, included stereo, newly excluded, re-included after each round) and stats (per round, the
        iteration statistics as optimize() returns them)."""
        n2 = np.array([len(f.omega2) for f in frames], np.int64); n3 = np.array([len(f.omega3) for f in frames], np.int64)
        ptr2 = np.concatenate([[0], np.cumsum(n2)]); ptr3 = np.concatenate([[0], np.cumsum(n3)])
        cat = lambda name, w: np.concatenate([np.asarray(getattr(f, name), np.float64).reshape(-1, w) for f in frames]) if frames else np.zeros((0, w))
        r = self.optimize_poses_flat(cat("q", 4), cat("t", 3), cat("cam", 5), ptr2, cat("X2", 3), cat("meas2", 2), cat("omega2", 1).ravel(),
                                     ptr3, cat("X3", 3), cat("meas3", 3), cat("omega3", 1).ravel(), rounds)
        off = np.concatenate([[0], np.cumsum([int(x.iterations) for x in rounds])])
        E2 = int(ptr2[-1])
        res = []
        for b in range(len(frames)):
            stats = []
            for k in range(len(rounds)):
                rows = r["stats"][b, off[k]:off[k] + r["nstats"][b, k]]
                stats.append([dict(iteration=int(s["iteration"]), trials=int(s["trials"]), chi2=float(s["chi2"]), lambda_=float(s["lambda_"]),
                                   pcg_iters=int(s["pcg_iters"]), pcg_failed=int(s["pcg_failed"])) for s in rows])
            res.append(dict(q=r["q"][b], t=r["t"][b], counts=r["counts"][b], stats=stats,
                            levels=np.concatenate([r["levels"][ptr2[b]:ptr2[b + 1]], r["levels"][E2 + ptr3[b]:E2 + ptr3[b + 1]]])))
        return res

    # --- batched Sim(3) alignment (ORB-SLAM2's OptimizeSim3 over many keyframe pairs in one launch) ------------------------------------
    def optimize_sim3_flat(self, ptr, q, t, s, cam1, cam2, fix_scale, X1, X2, obs1, obs2, omega1, omega2, params=None, B=None, N=None):
        """cuba_engine_optimize_sim3 on flat arrays (include/cuba_b200.h); fix_scale may be None; B / N default to the array sizes.
        Returns a dict of q [B,4], t [B,3], s [B], levels [N], ninliers [B], stats [B, iterations + max(bad, good)] (structured) and
        nstats [B,2]."""
        params = Sim3Params() if params is None else params
        f64 = lambda a, w: np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1, w) if w > 1 else np.asarray(a, dtype=np.float64).reshape(-1))
        q, t, s, cam1, cam2 = f64(q, 4), f64(t, 3), f64(s, 1), f64(cam1, 4), f64(cam2, 4)
        X1, X2, obs1, obs2, omega1, omega2 = f64(X1, 3), f64(X2, 3), f64(obs1, 2), f64(obs2, 2), f64(omega1, 1), f64(omega2, 1)
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
        st = np.frombuffer(out["stats"], dtype=np.dtype([("iteration", "<i4"), ("trials", "<i4"), ("chi2", "<f8"), ("lambda_", "<f8"),
                                                          ("pcg_iters", "<i4"), ("pcg_failed", "<i4")]))
        out["stats"] = st[:nb * S].reshape(nb, S).copy()
        return out

    def optimize_sim3(self, problems, params=None):
        """Refines S12 of every problem (graphio.Sim3Problem) under OptimizeSim3's schedule (Sim3Params) in one launch.  Returns, per
        problem, a dict of q [4], t [3], s, levels (0/1 per pair), ninliers and stats (the iteration statistics of the first and of
        the second optimize, as optimize() returns them)."""
        params = Sim3Params() if params is None else params
        n = np.array([len(p.omega1) for p in problems], np.int64)
        ptr = np.concatenate([[0], np.cumsum(n)])
        cat = lambda name, w: np.concatenate([np.asarray(getattr(p, name), np.float64).reshape(-1, w) for p in problems]) if problems else np.zeros((0, w))
        r = self.optimize_sim3_flat(ptr, cat("q", 4), cat("t", 3), cat("s", 1).ravel(), cat("cam1", 4), cat("cam2", 4),
                                    np.array([int(bool(p.fix_scale)) for p in problems], np.int32), cat("X1", 3), cat("X2", 3),
                                    cat("obs1", 2), cat("obs2", 2), cat("omega1", 1).ravel(), cat("omega2", 1).ravel(), params)
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
