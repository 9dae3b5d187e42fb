"""Graph files and the flat problem layout.

`.cubagraph` (little endian): magic b"CUBAGRF1", int64[4] = nposes, nlandmarks, nmono, nstereo, then
  pose_id i32[nP], pose_fixed i32[nP], q f64[nP,4] (x,y,z,w), t f64[nP,3], cam f64[nP,5] (fx,fy,cx,cy,bf),
  lm_id i32[nL], lm_fixed i32[nL], Xw f64[nL,3],
  mono_vP i32[nM], mono_vL i32[nM], mono_meas f64[nM,2], mono_info f64[nM],
  stereo_vP i32[nS], stereo_vL i32[nS], stereo_meas f64[nS,3], stereo_info f64[nS]
(vertex references in edges are vertex *ids*, like the reference's JSON: samples/sample_ba_from_file.cpp:93-157).

`flatten()` mirrors CudaBlockSolver::initialize (reference src/cuda_bundle_adjustment.cpp:115-261):
index assignment iP / iL in ascending id order, free vertices first, fixed appended; vertices without
edges skipped; edges with both ends fixed dropped; monocular edges get ids 0..E2-1, stereo E2..E2+E3-1.
The reference walks an unordered_set for the edges (order = heap addresses); we use file order.
"""
from __future__ import annotations

import dataclasses

import numpy as np

MAGIC = b"CUBAGRF1"

_FIELDS = (("pose_id", np.int32, 1), ("pose_fixed", np.int32, 1), ("q", np.float64, 4), ("t", np.float64, 3),
           ("cam", np.float64, 5), ("lm_id", np.int32, 1), ("lm_fixed", np.int32, 1), ("Xw", np.float64, 3),
           ("mono_vP", np.int32, 1), ("mono_vL", np.int32, 1), ("mono_meas", np.float64, 2), ("mono_info", np.float64, 1),
           ("stereo_vP", np.int32, 1), ("stereo_vL", np.int32, 1), ("stereo_meas", np.float64, 3),
           ("stereo_info", np.float64, 1))


def _count(name, n):
    if name.startswith("pose") or name in ("q", "t", "cam"):
        return n[0]
    if name.startswith("lm") or name == "Xw":
        return n[1]
    return n[2] if name.startswith("mono") else n[3]


def read_graph(path):
    with open(path, "rb") as f:
        if f.read(8) != MAGIC:
            raise ValueError("%s: not a cubagraph file" % path)
        n = np.fromfile(f, dtype=np.int64, count=4)
        g = {}
        for name, dt, width in _FIELDS:
            cnt = int(_count(name, n))
            a = np.fromfile(f, dtype=dt, count=cnt * width)
            g[name] = a.reshape(cnt, width) if width > 1 else a
    return g


def write_graph(path, g):
    with open(path, "wb") as f:
        f.write(MAGIC)
        np.array([len(g["pose_id"]), len(g["lm_id"]), len(g["mono_vP"]), len(g["stereo_vP"])], dtype=np.int64).tofile(f)
        for name, dt, _ in _FIELDS:
            np.ascontiguousarray(g[name], dtype=dt).tofile(f)


@dataclasses.dataclass
class FlatProblem:
    """Host-side flat problem = argument of cuba_engine_set_problem (include/cuba_b200.h)."""
    Pall: int
    numP: int
    Lall: int
    numL: int
    q: np.ndarray       # [Pall,4]
    t: np.ndarray       # [Pall,3]
    cam: np.ndarray     # [Pall,5]
    Xw: np.ndarray      # [Lall,3]
    idx2: np.ndarray    # [E2,2] int32 (iP,iL)
    meas2: np.ndarray   # [E2,2]
    omega2: np.ndarray  # [E2]
    idx3: np.ndarray    # [E3,2]
    meas3: np.ndarray   # [E3,3]
    omega3: np.ndarray  # [E3]
    # bookkeeping for writing results back into a graph dict
    pose_rows: np.ndarray = None   # row in graph["pose_id"] of each iP
    lm_rows: np.ndarray = None     # row in graph["lm_id"] of each iL
    mono_rows: np.ndarray = None   # row in graph mono arrays of each kept mono edge
    stereo_rows: np.ndarray = None

    @property
    def E2(self):
        return int(self.idx2.shape[0])

    @property
    def E3(self):
        return int(self.idx3.shape[0])

    @property
    def nedges(self):
        return self.E2 + self.E3

    def copy(self):
        return dataclasses.replace(self, **{f.name: (getattr(self, f.name).copy()
                                                     if isinstance(getattr(self, f.name), np.ndarray) else getattr(self, f.name))
                                            for f in dataclasses.fields(self)})


def _assign(ids, fixed, used):
    """free (ascending id) first, then fixed (ascending id); unused skipped. Returns rows in iX order, nfree."""
    order = np.argsort(ids, kind="stable")
    order = order[used[order]]
    free = order[fixed[order] == 0]
    fix = order[fixed[order] != 0]
    return np.concatenate([free, fix]).astype(np.int64), int(len(free))


def flatten(g) -> FlatProblem:
    pid, lid = g["pose_id"], g["lm_id"]
    pfix, lfix = g["pose_fixed"], g["lm_fixed"]
    # id -> row lookups (ids may be sparse)
    prow = {int(v): i for i, v in enumerate(pid)} if len(pid) and (pid.max() > 4 * len(pid) + 16) else None
    def rows_of(ids, table_ids, lut):
        if lut is not None:
            return np.array([lut[int(v)] for v in ids], dtype=np.int64)
        m = np.full(int(table_ids.max()) + 1 if len(table_ids) else 1, -1, dtype=np.int64)
        m[table_ids] = np.arange(len(table_ids))
        return m[ids]
    m_p = rows_of(g["mono_vP"], pid, prow); s_p = rows_of(g["stereo_vP"], pid, prow)
    m_l = rows_of(g["mono_vL"], lid, None); s_l = rows_of(g["stereo_vL"], lid, None)
    pused = np.zeros(len(pid), dtype=bool); lused = np.zeros(len(lid), dtype=bool)
    pused[m_p] = True; pused[s_p] = True; lused[m_l] = True; lused[s_l] = True
    prow_order, numP = _assign(pid, pfix, pused)
    lrow_order, numL = _assign(lid, lfix, lused)
    iP_of_row = np.full(len(pid), -1, dtype=np.int64); iP_of_row[prow_order] = np.arange(len(prow_order))
    iL_of_row = np.full(len(lid), -1, dtype=np.int64); iL_of_row[lrow_order] = np.arange(len(lrow_order))

    def edges(rp, rl, meas, info):
        keep = ~((pfix[rp] != 0) & (lfix[rl] != 0))
        rows = np.nonzero(keep)[0]
        idx = np.stack([iP_of_row[rp[rows]], iL_of_row[rl[rows]]], axis=1).astype(np.int32)
        return rows, np.ascontiguousarray(idx), np.ascontiguousarray(meas[rows], dtype=np.float64), \
            np.ascontiguousarray(info[rows], dtype=np.float64)

    mrows, idx2, meas2, om2 = edges(m_p, m_l, g["mono_meas"].reshape(-1, 2), g["mono_info"])
    srows, idx3, meas3, om3 = edges(s_p, s_l, g["stereo_meas"].reshape(-1, 3), g["stereo_info"])
    return FlatProblem(
        Pall=len(prow_order), numP=numP, Lall=len(lrow_order), numL=numL,
        q=np.ascontiguousarray(g["q"][prow_order], dtype=np.float64), t=np.ascontiguousarray(g["t"][prow_order], dtype=np.float64),
        cam=np.ascontiguousarray(g["cam"][prow_order], dtype=np.float64), Xw=np.ascontiguousarray(g["Xw"][lrow_order], dtype=np.float64),
        idx2=idx2.reshape(-1, 2), meas2=meas2.reshape(-1, 2), omega2=om2, idx3=idx3.reshape(-1, 2), meas3=meas3.reshape(-1, 3), omega3=om3,
        pose_rows=prow_order, lm_rows=lrow_order, mono_rows=mrows, stereo_rows=srows)


@dataclasses.dataclass
class PoseFrame:
    """One frame of Engine.optimize_poses: a free pose and its edges, each carrying its own world point, which is held fixed."""
    q: np.ndarray       # [4]
    t: np.ndarray       # [3]
    cam: np.ndarray     # [5]
    X2: np.ndarray      # [E2,3]
    meas2: np.ndarray   # [E2,2]
    omega2: np.ndarray  # [E2]
    X3: np.ndarray      # [E3,3]
    meas3: np.ndarray   # [E3,3]
    omega3: np.ndarray  # [E3]
    mono_ids: np.ndarray = None     # edge ids (0..E2-1) of the flat problem the frame was cut from
    stereo_ids: np.ndarray = None   # ids among the stereo edges (0..E3-1)

    def flat_problem(self, q=None, t=None, keep=None) -> FlatProblem:
        """The frame as a flat problem (its pose the only vertex, free; one fixed landmark per edge) at pose (q, t) (default: the
        frame's), with only the edges where keep[mono + stereo] is true (default: all): what the engine optimises for the frame."""
        E2 = len(self.omega2)
        keep = np.ones(E2 + len(self.omega3), bool) if keep is None else np.asarray(keep, bool)
        m, s = keep[:E2], keep[E2:]
        n2, n3 = int(m.sum()), int(s.sum())
        q = self.q if q is None else q
        t = self.t if t is None else t
        return FlatProblem(
            Pall=1, numP=1, Lall=n2 + n3, numL=0, q=np.array(q, dtype=np.float64).reshape(1, 4), t=np.array(t, dtype=np.float64).reshape(1, 3),
            cam=np.array(self.cam, dtype=np.float64).reshape(1, 5), Xw=np.concatenate([self.X2[m], self.X3[s]]).reshape(-1, 3),
            idx2=np.stack([np.zeros(n2), np.arange(n2)], 1).astype(np.int32), meas2=self.meas2[m].reshape(-1, 2), omega2=self.omega2[m],
            idx3=np.stack([np.zeros(n3), n2 + np.arange(n3)], 1).astype(np.int32), meas3=self.meas3[s].reshape(-1, 3), omega3=self.omega3[s])


def pose_frames(prob: FlatProblem, rows):
    """The frames of the poses `rows` (indices iP of prob): each pose with all of its edges in edge-id order, the edges' points taken
    from prob.Xw.  What flatten() gives for the graph of that one pose, free, with its edges and their landmarks, fixed."""
    def groups(idx):
        order = np.argsort(idx[:, 0], kind="stable")
        ptr = np.searchsorted(idx[order, 0], np.arange(prob.Pall + 1))
        return order, ptr
    o2, p2 = groups(prob.idx2)
    o3, p3 = groups(prob.idx3)
    out = []
    for p in rows:
        p = int(p)
        m = o2[p2[p]:p2[p + 1]]; s = o3[p3[p]:p3[p + 1]]
        out.append(PoseFrame(q=prob.q[p].copy(), t=prob.t[p].copy(), cam=prob.cam[p].copy(),
                             X2=prob.Xw[prob.idx2[m, 1]], meas2=prob.meas2[m].copy(), omega2=prob.omega2[m].copy(),
                             X3=prob.Xw[prob.idx3[s, 1]], meas3=prob.meas3[s].copy(), omega3=prob.omega3[s].copy(),
                             mono_ids=m, stereo_ids=s))
    return out


def _cat(items, name, w):
    """the field `name` of every item as one contiguous float64 array [n, w] ([n] for w = 1)"""
    a = np.concatenate([np.asarray(getattr(x, name), np.float64).reshape(-1, w) for x in items]) if items else np.zeros((0, w))
    return np.ascontiguousarray(a.ravel() if w == 1 else a)


def _ptr(counts):
    return np.concatenate([[0], np.cumsum(np.asarray(counts, np.int64))]).astype(np.int32)


def pose_batch_arrays(frames):
    """the flat arrays of cuba_pose_batch for a list of PoseFrame: the keyword arguments of Engine.optimize_poses_flat (numpy) and,
    moved to the GPU, of Engine.optimize_poses_device"""
    return dict(q=_cat(frames, "q", 4), t=_cat(frames, "t", 3), cam=_cat(frames, "cam", 5), ptr2=_ptr([len(f.omega2) for f in frames]),
                X2=_cat(frames, "X2", 3), meas2=_cat(frames, "meas2", 2), omega2=_cat(frames, "omega2", 1),
                ptr3=_ptr([len(f.omega3) for f in frames]), X3=_cat(frames, "X3", 3), meas3=_cat(frames, "meas3", 3),
                omega3=_cat(frames, "omega3", 1))


@dataclasses.dataclass
class PointBatch:
    """The points of Engine.optimize_points: a table of P poses, held fixed, and B points, each an initial position and its edges
    (mono [ptr2[b], ptr2[b+1]), stereo [ptr3[b], ptr3[b+1])), each edge naming its pose by index in the table."""
    q: np.ndarray       # [P,4] x,y,z,w
    t: np.ndarray       # [P,3]
    cam: np.ndarray     # [P,5]
    Xw: np.ndarray      # [B,3]
    ptr2: np.ndarray    # [B+1] int32
    iP2: np.ndarray     # [E2] int32
    meas2: np.ndarray   # [E2,2]
    omega2: np.ndarray  # [E2]
    ptr3: np.ndarray    # [B+1] int32
    iP3: np.ndarray     # [E3] int32
    meas3: np.ndarray   # [E3,3]
    omega3: np.ndarray  # [E3]
    landmarks: np.ndarray = None    # [B] landmark ids (iL) of the flat problem the points were cut from
    mono_ids: np.ndarray = None     # [E2] edge ids (0..E2-1) of that flat problem
    stereo_ids: np.ndarray = None   # [E3] ids among its stereo edges

    @property
    def B(self):
        return len(self.ptr2) - 1

    def arrays(self):
        """the keyword arguments of Engine.optimize_points_flat (numpy) and, moved to the GPU, of Engine.optimize_points_device"""
        return {k: getattr(self, k) for k in ("Xw", "q", "t", "cam", "ptr2", "iP2", "meas2", "omega2", "ptr3", "iP3", "meas3", "omega3")}

    def sub_problem(self, b, Xw=None, keep=None) -> FlatProblem:
        """The engine's sub-problem of point b: the poses its kept edges name (ascending table index) as fixed vertices, the point at Xw
        (default: its input position) as the only free landmark, and the edges where keep[mono + stereo] is true (default: all)."""
        m = np.arange(self.ptr2[b], self.ptr2[b + 1]); s = np.arange(self.ptr3[b], self.ptr3[b + 1])
        keep = np.ones(len(m) + len(s), bool) if keep is None else np.asarray(keep, bool)
        m, s = m[keep[:len(m)]], s[keep[len(m):]]
        poses, inv = np.unique(np.concatenate([self.iP2[m], self.iP3[s]]), return_inverse=True)
        ip = inv.astype(np.int32)
        X = self.Xw[b] if Xw is None else Xw
        return FlatProblem(
            Pall=len(poses), numP=0, Lall=1, numL=1, q=self.q[poses].reshape(-1, 4).copy(), t=self.t[poses].reshape(-1, 3).copy(),
            cam=self.cam[poses].reshape(-1, 5).copy(), Xw=np.array(X, dtype=np.float64).reshape(1, 3),
            idx2=np.stack([ip[:len(m)], np.zeros(len(m), np.int32)], 1).astype(np.int32), meas2=self.meas2[m].reshape(-1, 2),
            omega2=self.omega2[m].copy(), idx3=np.stack([ip[len(m):], np.zeros(len(s), np.int32)], 1).astype(np.int32),
            meas3=self.meas3[s].reshape(-1, 3), omega3=self.omega3[s].copy())


def point_batch(prob: FlatProblem, landmarks) -> PointBatch:
    """The points of the landmarks (indices iL of prob) against prob's whole pose table: each landmark at prob.Xw with all of its
    edges in edge-id order.  Point b's sub_problem is what flatten() gives for the graph of that one landmark, free, with its edges
    and their poses, fixed."""
    def groups(idx):
        order = np.argsort(idx[:, 1], kind="stable")
        return order, np.searchsorted(idx[order, 1], np.arange(prob.Lall + 1))
    o2, p2 = groups(prob.idx2)
    o3, p3 = groups(prob.idx3)
    L = np.asarray(landmarks, np.int64).reshape(-1)
    m = np.concatenate([o2[p2[l]:p2[l + 1]] for l in L]).astype(np.int64) if len(L) else np.zeros(0, np.int64)
    s = np.concatenate([o3[p3[l]:p3[l + 1]] for l in L]).astype(np.int64) if len(L) else np.zeros(0, np.int64)
    return PointBatch(
        q=np.ascontiguousarray(prob.q, dtype=np.float64).reshape(-1, 4), t=np.ascontiguousarray(prob.t, dtype=np.float64).reshape(-1, 3),
        cam=np.ascontiguousarray(prob.cam, dtype=np.float64).reshape(-1, 5), Xw=np.ascontiguousarray(prob.Xw[L], dtype=np.float64).reshape(-1, 3),
        ptr2=_ptr(p2[L + 1] - p2[L]), iP2=np.ascontiguousarray(prob.idx2[m, 0], dtype=np.int32),
        meas2=np.ascontiguousarray(prob.meas2[m], dtype=np.float64).reshape(-1, 2), omega2=np.ascontiguousarray(prob.omega2[m], dtype=np.float64),
        ptr3=_ptr(p3[L + 1] - p3[L]), iP3=np.ascontiguousarray(prob.idx3[s, 0], dtype=np.int32),
        meas3=np.ascontiguousarray(prob.meas3[s], dtype=np.float64).reshape(-1, 3), omega3=np.ascontiguousarray(prob.omega3[s], dtype=np.float64),
        landmarks=L, mono_ids=m, stereo_ids=s)


@dataclasses.dataclass
class Sim3Problem:
    """One problem of Engine.optimize_sim3 (ORB-SLAM2's OptimizeSim3): S12 = (q, t, s), S12 X = s R(q) X + t, from camera 2 into
    camera 1, and N matched pairs: X1 / X2 the point in camera-1 / camera-2 coordinates, obs1 / obs2 its keypoints, omega1 / omega2
    their scalar informations."""
    q: np.ndarray       # [4] x,y,z,w
    t: np.ndarray       # [3]
    s: float
    cam1: np.ndarray    # [4] fx,fy,cx,cy
    cam2: np.ndarray    # [4]
    X1: np.ndarray      # [N,3]
    X2: np.ndarray      # [N,3]
    obs1: np.ndarray    # [N,2]
    obs2: np.ndarray    # [N,2]
    omega1: np.ndarray  # [N]
    omega2: np.ndarray  # [N]
    fix_scale: bool = False
    landmarks: np.ndarray = None   # [N] landmark ids (iL) of the flat problem the pairs were cut from


def _rotation(q):
    x, y, z, w = (float(v) for v in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _quaternion(R):
    """the unit quaternion (x, y, z, w), w >= 0, of a rotation matrix"""
    K = np.array([[R[0, 0] - R[1, 1] - R[2, 2], R[1, 0] + R[0, 1], R[2, 0] + R[0, 2], R[2, 1] - R[1, 2]],
                  [R[1, 0] + R[0, 1], R[1, 1] - R[0, 0] - R[2, 2], R[2, 1] + R[1, 2], R[0, 2] - R[2, 0]],
                  [R[2, 0] + R[0, 2], R[2, 1] + R[1, 2], R[2, 2] - R[0, 0] - R[1, 1], R[1, 0] - R[0, 1]],
                  [R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1], R[0, 0] + R[1, 1] + R[2, 2]]]) / 3
    w, v = np.linalg.eigh(K)
    q = v[:, np.argmax(w)]
    return q if q[3] >= 0 else -q


def sim3_problems(prob: FlatProblem, pairs, scale=1.0, fix_scale=False):
    """The Sim3 problems of the pose pairs (i, j) (indices iP of prob): one matched pair per landmark both poses observe, in landmark
    order; obs = (u, v) of the pose's edge to the landmark, (u_left, v) for a stereo edge (the first edge in edge-id order where a
    pose has several); X1 / X2 = the landmark's point in camera i / camera j, X2 divided by the pair's scale drift s0 (`scale`: one
    value, or one per pair).  S12 is set to the planted value (R_i R_j^T, t_i - R_i R_j^T t_j, s0), which maps X2 onto X1 exactly."""
    P = np.concatenate([prob.idx2[:, 0], prob.idx3[:, 0]]).astype(np.int64)
    L = np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]]).astype(np.int64)
    uv = np.concatenate([np.asarray(prob.meas2).reshape(-1, 2), np.asarray(prob.meas3).reshape(-1, 3)[:, :2]])
    om = np.concatenate([prob.omega2, prob.omega3])
    order = np.lexsort((np.arange(len(P)), L, P))
    P, L, uv, om = P[order], L[order], uv[order], om[order]
    first = np.ones(len(P), bool)
    first[1:] = (P[1:] != P[:-1]) | (L[1:] != L[:-1])
    P, L, uv, om = P[first], L[first], uv[first], om[first]
    ptr = np.searchsorted(P, np.arange(prob.Pall + 1))
    pairs = [(int(i), int(j)) for i, j in pairs]
    s0 = np.broadcast_to(np.asarray(scale, dtype=np.float64), (len(pairs),))
    out = []
    for k, (i, j) in enumerate(pairs):
        common, a, b = np.intersect1d(L[ptr[i]:ptr[i + 1]], L[ptr[j]:ptr[j + 1]], assume_unique=True, return_indices=True)
        a, b = a + ptr[i], b + ptr[j]
        Ri, Rj = _rotation(prob.q[i]), _rotation(prob.q[j])
        X = np.asarray(prob.Xw)[common].reshape(-1, 3)
        R12 = Ri @ Rj.T
        out.append(Sim3Problem(
            q=_quaternion(R12), t=prob.t[i] - R12 @ prob.t[j], s=float(s0[k]), cam1=np.array(prob.cam[i][:4], dtype=np.float64),
            cam2=np.array(prob.cam[j][:4], dtype=np.float64), X1=X @ Ri.T + prob.t[i], X2=(X @ Rj.T + prob.t[j]) / s0[k],
            obs1=uv[a].copy(), obs2=uv[b].copy(), omega1=om[a].copy(), omega2=om[b].copy(), fix_scale=bool(fix_scale), landmarks=common))
    return out


def sim3_batch_arrays(problems):
    """the flat arrays of cuba_sim3_batch for a list of Sim3Problem, fix_scale from each problem: the keyword arguments of
    Engine.optimize_sim3_flat (numpy) and, moved to the GPU, of Engine.optimize_sim3_device"""
    return dict(ptr=_ptr([len(p.omega1) for p in problems]), q=_cat(problems, "q", 4), t=_cat(problems, "t", 3),
                s=_cat(problems, "s", 1), cam1=_cat(problems, "cam1", 4), cam2=_cat(problems, "cam2", 4),
                fix_scale=np.array([int(bool(p.fix_scale)) for p in problems], np.int32), X1=_cat(problems, "X1", 3),
                X2=_cat(problems, "X2", 3), obs1=_cat(problems, "obs1", 2), obs2=_cat(problems, "obs2", 2), omega1=_cat(problems, "omega1", 1),
                omega2=_cat(problems, "omega2", 1))


def write_back(g, prob: FlatProblem, q, t, Xw):
    """finalize(): reference src/cuda_bundle_adjustment.cpp:512-526 (fixed vertices are written back too)."""
    g["q"][prob.pose_rows] = q
    g["t"][prob.pose_rows] = t
    g["Xw"][prob.lm_rows] = Xw
