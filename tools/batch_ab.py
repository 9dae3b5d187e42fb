#!/usr/bin/env python3
"""Every output of the batched LM kernels on the workloads of tools/pose_batch_timing.py and tools/sim3_batch_timing.py, so that two
builds of the library can be compared bit for bit (swap the in-tree library between two `dump` runs, as tools/ab_libs.sh does):

  dump OUT.npz        Engine.optimize_poses on every frame of ba_kitti_00 (kitti00_shaped when the fixture is absent) under
                      ORB-SLAM2's schedule, Engine.optimize_sim3 on the Sim3 workload with fix_scale off and on, and
                      Engine.optimize_points on every landmark (perturbed) under tools/point_batch_timing.py's schedule: q, t, s, Xw,
                      levels, counts / ninliers, nstats and the per-iteration statistics (iteration, trials, chi2, lambda)
  compare A.npz B.npz the bytes, dtype and shape of every array; prints the arrays that differ and exits 1 if any does

Usage: python tools/batch_ab.py dump out.npz;  python tools/batch_ab.py compare a.npz b.npz"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
import point_batch_timing  # noqa: E402
import sim3_batch_timing  # noqa: E402


def flatten(prefix, res):
    """the per-problem result dicts of optimize_poses / optimize_sim3 as flat arrays"""
    out = {}
    for key in res[0]:
        if key == "stats":
            rows = [s for r in res for rnd in r["stats"] for s in rnd]
            out[prefix + "nstats"] = np.array([len(rnd) for r in res for rnd in r["stats"]], np.int64)
            for f in ("iteration", "trials", "chi2", "lambda_", "pcg_iters", "pcg_failed"):
                out[prefix + "stats_" + f] = np.array([s[f] for s in rows])
        else:
            out[prefix + key] = np.concatenate([np.atleast_1d(np.asarray(r[key])).ravel() for r in res])
    return out


def dump(path):
    pkg = ge.load_package()
    fx = os.path.join(ROOT, "oracle", "_ref", "fixtures", "ba_kitti_00.cubagraph")
    g = pkg.graphio.read_graph(fx) if os.path.exists(fx) else pkg.synth.make_config("kitti00_shaped")
    prob = pkg.graphio.flatten(g)
    eng = pkg.Engine(device=0)
    arrays = flatten("pose_", eng.optimize_poses(pkg.graphio.pose_frames(prob, range(prob.Pall)), pkg.orbslam2_pose_schedule()))
    problems = sim3_batch_timing.workload(pkg, prob, 5)
    for fix in (False, True):
        for p in problems:
            p.fix_scale = fix
        arrays.update(flatten("sim3_fix%d_" % fix, eng.optimize_sim3(problems)))
    pts = prob.copy()
    pts.Xw = pts.Xw + np.random.default_rng(7).normal(0, 0.1, pts.Xw.shape)
    arrays.update(flatten("points_", eng.optimize_points(pkg.graphio.point_batch(pts, range(pts.Lall)), point_batch_timing.schedule(pkg))))
    np.savez(path, **arrays)
    print("%s: %d frames, %d Sim3 problems, %d arrays" % (path, prob.Pall, len(problems), len(arrays)))


def compare(a, b):
    A, B = np.load(a), np.load(b)
    same = lambda x, y: x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
    bad = sorted(k for k in set(A.files) | set(B.files) if k not in A.files or k not in B.files or not same(A[k], B[k]))
    for k in bad:
        print("DIFFERENT:", k)
    print("%d arrays, %d different" % (len(set(A.files) | set(B.files)), len(bad)))
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "dump":
        dump(sys.argv[2])
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    else:
        sys.exit(__doc__)
