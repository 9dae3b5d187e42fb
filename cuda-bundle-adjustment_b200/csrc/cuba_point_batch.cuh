// cuba_point_batch.cuh -- structure-only refinement of many map points in one launch (g2o's StructureOnlySolver, SVO's structure
// optimisation, the refinement ORB-SLAM2's CreateNewMapPoints leaves out).
//
// A point is one free world position and its monocular / stereo edges, each naming a pose of a shared table; the poses are held fixed.
// k_point_batch runs one WARP per point over the whole round schedule: per round an optional restart from the input position, the
// LM loop of Engine::optimize at warp level (lm::optimize_warp, cuba_lm_batch.cuh) and the outlier test of lv::k_classify_edges on the
// committed position.  A landmark has a handful of edges (4.2 on average on ba_kitti_00), so a CTA per point would leave most of
// its threads idle and pay two barriers per sum; a warp sums with shuffles alone and needs no barrier at all.
//
// Per LM iteration the lanes stride over the point's edges at level 0 and accumulate the 6 unique Hll entries, bl and the robust
// chi2 (the formulas of k_linearize_landmark); the damped 3x3 solve is the engine's landmark-only arithmetic (sym3_inverse of
// Hll + lambda I as in k_inv_hll, x = inv bl in k_solve_landmarks_only's order) and the update Xw + x.
//
// Edges and their pose records are read from global memory on every pass; levels live in global memory, one byte per edge, and a
// lane reads and writes only its own edges (k = lane mod 32), so no fence is needed between passes.
//
// The per-point problem (Point) reads its edges through an edge source: BatchEdges here, the engine's landmark-major stream in
// k_refine_landmarks (cuba_landmark_refine.cuh), which runs the same rounds (run_schedule) on the engine's own landmarks.
#pragma once

#include "cuba_lm_batch.cuh"
#include "cuba_pose_batch.cuh"

namespace cuba_b200 {
namespace ptb {

constexpr int WARPS = lm::BLOCK / 32;  // points per CTA

struct Args {
	int B;
	const double* Xw;                 // [B][4]  X pad
	const double* pose;               // [P][8]  q(x,y,z,w) t pad
	const double* cam;                // [P][8]  fx fy cx cy bf pad
	const double* edge;               // [E][4]  meas(3) omega; point b: ptr2[b]+ptr3[b] .., its mono edges first (meas[2] = 0)
	const int* iP;                    // [E]     pose of each edge, order of `edge`
	const int* ptr2;                  // [B+1]
	const int* ptr3;                  // [B+1]
	double* XwOut;                    // [B][4]
	unsigned char* level;             // [E], order of `edge`
	int* counts;                      // [B][n][4]
	int* nstats;                      // [B][n]
	lm::IterStat* stats;              // [B][statOff[n]] or null
};

// The edges of a point of the batch: point b's are e0 .. e0 + n of the packed arrays, its mono edges first
struct BatchEdges {
	const double* edge;               // Args::edge, iP, level
	const int* iP;
	unsigned char* level;
	int e0, nMono;

	// edge k's pose and type
	__device__ __forceinline__ int pose(int k, bool& stereo) const { stereo = k >= nMono; return iP[e0 + k]; }
	// edge k's measurement (m[2] = 0 for a mono edge) and omega
	__device__ __forceinline__ void meas(int k, bool, double m[3], double& om) const
	{
		ld2(edge + 4 * (size_t)(e0 + k), m[0], m[1]);
		ld2(edge + 4 * (size_t)(e0 + k) + 2, m[2], om);
	}
	// edge k's level byte
	__device__ __forceinline__ unsigned char* slot(int k) const { return level + e0 + k; }
};

// one point's LM problem under a round's robust kernels, over the edges of an edge source (BatchEdges; StreamEdges of
// cuba_landmark_refine.cuh); the state is X(3), the same in every lane
template <class Edges>
struct Point {
	static constexpr int N = 3;
	const double* pose;               // [P][8] q t pad, [P][8] fx fy cx cy bf pad
	const double* cam;
	Edges ed;
	int n;
	RobustParams rk;

	// edge k's pose, type, camera-frame point and residual at X, and its weighted squared error om |r|^2
	__device__ __forceinline__ double residual(int k, const double X[3], bool& stereo, double q[4], double c[5], double Xc[3], double r[3],
		double& om) const
	{
		double t[3], m[3];
		load_pose(pose, cam, ed.pose(k, stereo), q, t, c);
		ed.meas(k, stereo, m, om);
		edge_residual(q, t, c, X, m, stereo, Xc, r);
		return om * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
	}

	// Hll (upper, packed) += w JL^T JL, bl += w JL^T r and the robust chi2 of the edges at level 0
	__device__ __forceinline__ void linearize(double acc[10], const double* X) const
	{
		for (int k = threadIdx.x & 31; k < n; k += 32) {
			if (*ed.slot(k)) continue;
			bool stereo;
			double q[4], c[5], Xc[3], r[3], om, rho, drho;
			const double e2 = residual(k, X, stereo, q, c, Xc, r, om);
			// constant indices: a run-time index into rk would keep the whole Point in local memory
			robust<double>(stereo ? rk.type[1] : rk.type[0], stereo ? rk.delta[1] : rk.delta[0], e2, rho, drho);
			acc[9] += rho;
			const double w = om * drho;
			double JP[3][6], JL[3][3], wJL[3][3], wr[3];
			edge_jacobians(q, c, Xc, stereo, JP, JL);
#pragma unroll
			for (int mm = 0; mm < 3; mm++) {
				wr[mm] = w * r[mm];
#pragma unroll
				for (int l = 0; l < 3; l++) wJL[mm][l] = w * JL[mm][l];
			}
			// k_linearize_landmark's entries 00, 01, 02, 11, 12, 22, bl, in the packed order 00, 01, 11, 02, 12, 22
			acc[0] += JL[0][0] * wJL[0][0] + JL[1][0] * wJL[1][0] + JL[2][0] * wJL[2][0];
			acc[1] += JL[0][0] * wJL[0][1] + JL[1][0] * wJL[1][1] + JL[2][0] * wJL[2][1];
			acc[3] += JL[0][0] * wJL[0][2] + JL[1][0] * wJL[1][2] + JL[2][0] * wJL[2][2];
			acc[2] += JL[0][1] * wJL[0][1] + JL[1][1] * wJL[1][1] + JL[2][1] * wJL[2][1];
			acc[4] += JL[0][1] * wJL[0][2] + JL[1][1] * wJL[1][2] + JL[2][1] * wJL[2][2];
			acc[5] += JL[0][2] * wJL[0][2] + JL[1][2] * wJL[1][2] + JL[2][2] * wJL[2][2];
			acc[6] += JL[0][0] * wr[0] + JL[1][0] * wr[1] + JL[2][0] * wr[2];
			acc[7] += JL[0][1] * wr[0] + JL[1][1] * wr[1] + JL[2][1] * wr[2];
			acc[8] += JL[0][2] * wr[0] + JL[1][2] * wr[1] + JL[2][2] * wr[2];
		}
	}

	// robust chi2 of the edges at level 0
	__device__ __forceinline__ double chi2(const double* X) const
	{
		double chi = 0;
		for (int k = threadIdx.x & 31; k < n; k += 32) {
			if (*ed.slot(k)) continue;
			bool stereo;
			double q[4], c[5], Xc[3], r[3], om, rho, drho;
			const double e2 = residual(k, X, stereo, q, c, Xc, r, om);
			robust<double>(stereo ? rk.type[1] : rk.type[0], stereo ? rk.delta[1] : rk.delta[0], e2, rho, drho);
			chi += rho;
		}
		return chi;
	}

	// the engine's landmark-only solve: sym3_inverse of Hll + lambda I (k_inv_hll), x = inv bl (k_solve_landmarks_only).  A singular
	// system gives a non-finite x, whose trial the gain ratio rejects.
	__device__ __forceinline__ void solve(const double sys[10], double lambda, double x[3]) const
	{
		double B[6];
		sym3_inverse<double>(sys[0] + lambda, sys[1], sys[3], sys[2] + lambda, sys[4], sys[5] + lambda, B);
		x[0] = B[0] * sys[6] + B[1] * sys[7] + B[2] * sys[8];
		x[1] = B[1] * sys[6] + B[3] * sys[7] + B[4] * sys[8];
		x[2] = B[2] * sys[6] + B[4] * sys[7] + B[5] * sys[8];
	}

	__device__ __forceinline__ void update(const double x[3], const double* X, double* Xt) const
	{
#pragma unroll
		for (int i = 0; i < 3; i++) Xt[i] = X[i] + x[i];
	}

	// the outlier test of lv::k_classify_edges on X: new levels, and the warp's counts (included mono, included stereo, newly
	// excluded, re-included) in every lane.  A lane reads and writes only its own edges' levels.
	__device__ __forceinline__ void classify(const double X[3], const pb::Round& R, int c4[4]) const
	{
		c4[0] = c4[1] = c4[2] = c4[3] = 0;
		for (int k = threadIdx.x & 31; k < n; k += 32) {
			bool stereo;
			double q[4], c[5], Xc[3], r[3], om;
			const double chi2 = residual(k, X, stereo, q, c, Xc, r, om);
			const bool fail = chi2 > (stereo ? R.chi2[1] : R.chi2[0]) || ((R.flags & lv::FAIL_DEPTH) && Xc[2] <= 0);
			unsigned char* s = ed.slot(k);
			const int old = *s;
			const int now = (R.flags & lv::REINCLUDE) ? (fail ? 1 : 0) : (old | (fail ? 1 : 0));
			if (now != old) *s = (unsigned char)now;
			c4[0] += !now && !stereo; c4[1] += !now && stereo; c4[2] += !old && now; c4[3] += old && !now;
		}
#pragma unroll
		for (int k = 0; k < 4; k++)
#pragma unroll
			for (int o = 16; o > 0; o >>= 1) c4[k] += __shfl_xor_sync(0xffffffffu, c4[k], o);
	}
};

// The round schedule on one point, by its warp: per round an optional restart to Xin, lm::optimize_warp from X, then the outlier
// test on the committed X.  included: the point's edges at level 0 on entry.  stats: the point's first stat slot, or null.  After
// each round, out(rd, iterations written, c4) with the warp's counts in every lane.
template <class Edges, class Out>
__device__ __forceinline__ void run_schedule(const double* pose, const double* cam, const Edges& ed, int n, const pb::Schedule& s,
	const double Xin[3], double X[3], int included, lm::IterStat* stats, Out&& out)
{
	for (int rd = 0; rd < s.n; rd++) {
		const pb::Round R = s.r[rd];
		if (R.restart)
#pragma unroll
			for (int i = 0; i < 3; i++) X[i] = Xin[i];
		const Point<Edges> P = { pose, cam, ed, n, s.rk[rd] };
		const int nIt = lm::optimize_warp(P, X, included, R.iterations, stats ? stats + s.statOff[rd] : nullptr);
		int c4[4];
		P.classify(X, R, c4);
		included = c4[0] + c4[1];
		out(rd, nIt, c4);
	}
}

__global__ void __launch_bounds__(lm::BLOCK) k_point_batch(const Args a, const pb::Schedule s)
{
	const int b = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
	if (b >= a.B) return;
	const int e0 = a.ptr2[b] + a.ptr3[b];
	const int nMono = a.ptr2[b + 1] - a.ptr2[b];
	const int n = nMono + a.ptr3[b + 1] - a.ptr3[b];
	double Xin[3], X[3];
#pragma unroll
	for (int i = 0; i < 3; i++) X[i] = Xin[i] = a.Xw[4 * (size_t)b + i];
	for (int k = lane; k < n; k += 32) a.level[e0 + k] = 0;
	const BatchEdges ed = { a.edge, a.iP, a.level, e0, nMono };
	run_schedule(a.pose, a.cam, ed, n, s, Xin, X, n, a.stats ? a.stats + (size_t)b * s.statOff[s.n] : nullptr,
		[&](int rd, int nIt, const int c4[4]) {
			if (lane < 4) a.counts[((size_t)b * s.n + rd) * 4 + lane] = lane == 0 ? c4[0] : lane == 1 ? c4[1] : lane == 2 ? c4[2] : c4[3];
			if (lane == 0) a.nstats[(size_t)b * s.n + rd] = nIt;
		});
	if (lane < 4) a.XwOut[4 * (size_t)b + lane] = lane == 0 ? X[0] : lane == 1 ? X[1] : lane == 2 ? X[2] : 0.0;
}

}  // namespace ptb
}  // namespace cuba_b200
