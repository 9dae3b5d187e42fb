// cuba_pose_batch.cuh -- pose optimisation of many frames in one launch (ORB-SLAM2's Optimizer::PoseOptimization, batched).
//
// A frame is one free SE(3) pose and its monocular / stereo edges, each with its own world point held fixed.  k_pose_batch runs one
// CTA per frame over the whole round schedule: per round an optional restart from the input pose, the LM loop of Engine::optimize
// (lm::optimize, cuba_lm_batch.cuh) and the outlier test of lv::k_classify_edges on the committed pose.  Nothing leaves the CTA
// between rounds; the host reads the results once, after the launch.
//
// Per LM iteration a block-stride pass over the frame's edges at level 0 accumulates the 21 unique Hpp entries, bp and the robust
// chi2 (the formulas of k_linearize_pose); the damped 6x6 solve is k_solve_poses_only's and the update se3_update.
//
// Edges are read from global memory on every pass (a frame of ~400 edges is 26 KB and stays in L1/L2); levels live in global
// memory, one byte per edge.
#pragma once

#include "cuba_lm_batch.cuh"

namespace cuba_b200 {
namespace pb {

constexpr int MAX_ROUNDS = 8;         // include/cuba_b200.h: CUBA_POSE_MAX_ROUNDS

struct Round {
	int iterations;
	int restart;
	int flags;                        // lv::FAIL_DEPTH | lv::REINCLUDE
	double chi2[2];                   // test thresholds, mono / stereo
};
struct Schedule {
	int n;
	Round r[MAX_ROUNDS];
	RobustParams rk[MAX_ROUNDS];
	int statOff[MAX_ROUNDS + 1];      // first stat slot of each round within a frame; statOff[n] = slots per frame
};

struct Args {
	int B;
	const double* pose;               // [B][8]  q(x,y,z,w) t pad
	const double* cam;                // [B][8]  fx fy cx cy bf pad
	const double* edge;               // [E][8]  X(3) meas(3) omega pad; frame b: ptr2[b]+ptr3[b] .. , its mono edges first
	const int* ptr2;                  // [B+1]
	const int* ptr3;                  // [B+1]
	double* poseOut;                  // [B][8]
	unsigned char* level;             // [E], order of `edge`
	int* counts;                      // [B][n][4]
	int* nstats;                      // [B][n]
	lm::IterStat* stats;              // [B][statOff[n]] or null
};

__device__ __forceinline__ void load_edge(const double* __restrict__ p, double X[3], double m[3], double& om)
{
	ld2(p, X[0], X[1]); ld2(p + 2, X[2], m[0]); ld2(p + 4, m[1], m[2]);
	double pad;
	ld2(p + 6, om, pad);
}

// one frame's LM problem under a round's robust kernels; the state is the pose q(4) t(3) pad
struct Frame {
	static constexpr int N = 6;
	const double* edge;               // Args::edge, Args::level; the frame's edges are e0 .. e0 + n, mono first
	const unsigned char* level;
	int e0, n, nMono;
	const double* cam;                // shared memory
	RobustParams rk;

	__device__ __forceinline__ void load(const double* S, double q[4], double t[3], double c[5]) const
	{
#pragma unroll
		for (int i = 0; i < 4; i++) q[i] = S[i];
#pragma unroll
		for (int i = 0; i < 3; i++) t[i] = S[4 + i];
#pragma unroll
		for (int i = 0; i < 5; i++) c[i] = cam[i];
	}

	// edge k's residual at (q, t) and its robust chi2 rho(om |r|^2)
	__device__ __forceinline__ void residual(int k, const double q[4], const double t[3], const double c[5], double Xc[3], double r[3],
		double& om, double& rho, double& drho) const
	{
		const bool stereo = k >= nMono;
		double X[3], m[3];
		load_edge(edge + 8 * (size_t)(e0 + k), X, m, om);
		if (!stereo) m[2] = 0;
		edge_residual(q, t, c, X, m, stereo, Xc, r);
		const double e2 = om * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
		// constant indices: a run-time index into rk would keep the whole Frame in local memory
		robust<double>(stereo ? rk.type[1] : rk.type[0], stereo ? rk.delta[1] : rk.delta[0], e2, rho, drho);
	}

	// Hpp (upper, packed) += w JP^T JP, bp += w JP^T r and the robust chi2 of the edges at level 0
	__device__ __forceinline__ void linearize(double acc[28], const double* S) const
	{
		double q[4], t[3], c[5];
		load(S, q, t, c);
		for (int k = threadIdx.x; k < n; k += lm::BLOCK) {
			if (level[e0 + k]) continue;
			double Xc[3], r[3], om, rho, drho;
			residual(k, q, t, c, Xc, r, om, rho, drho);
			acc[27] += rho;
			const double w = om * drho;
			double JP[3][6], JL[3][3], wJP[3][6];
			edge_jacobians(q, c, Xc, k >= nMono, JP, JL);
#pragma unroll
			for (int mm = 0; mm < 3; mm++)
#pragma unroll
				for (int l = 0; l < 6; l++) wJP[mm][l] = w * JP[mm][l];
			int kk = 0;
#pragma unroll
			for (int cn = 0; cn < 6; cn++)
#pragma unroll
				for (int l = 0; l <= cn; l++) {
					acc[kk] += JP[0][l] * wJP[0][cn] + JP[1][l] * wJP[1][cn] + JP[2][l] * wJP[2][cn];
					kk++;
				}
#pragma unroll
			for (int l = 0; l < 6; l++) acc[21 + l] += wJP[0][l] * r[0] + wJP[1][l] * r[1] + wJP[2][l] * r[2];
		}
	}

	// robust chi2 of the edges at level 0
	__device__ __forceinline__ double chi2(const double* S) const
	{
		double q[4], t[3], c[5];
		load(S, q, t, c);
		double chi = 0;
		for (int k = threadIdx.x; k < n; k += lm::BLOCK) {
			if (level[e0 + k]) continue;
			double Xc[3], r[3], om, rho, drho;
			residual(k, q, t, c, Xc, r, om, rho, drho);
			chi += rho;
		}
		return chi;
	}

	// the SE(3) update of k_update_poses
	__device__ __forceinline__ void update(const double x[6], const double* S, double* St) const
	{
		double qq[4], tt[3];
		for (int i = 0; i < 4; i++) qq[i] = S[i];
		for (int i = 0; i < 3; i++) tt[i] = S[4 + i];
		se3_update(x, qq, tt);
		for (int i = 0; i < 4; i++) St[i] = qq[i];
		for (int i = 0; i < 3; i++) St[4 + i] = tt[i];
	}
};

__global__ void __launch_bounds__(lm::BLOCK) k_pose_batch(const Args a, const Schedule s)
{
	__shared__ lm::Shared<Frame::N> sh;
	__shared__ double s_in[8], s_cam[8];

	const int b = blockIdx.x, tid = threadIdx.x;
	const int e0 = a.ptr2[b] + a.ptr3[b];
	const int nMono = a.ptr2[b + 1] - a.ptr2[b];
	const int n = nMono + a.ptr3[b + 1] - a.ptr3[b];
	if (tid < 8) {
		s_in[tid] = a.pose[8 * (size_t)b + tid];
		s_cam[tid] = a.cam[8 * (size_t)b + tid];
		sh.state[0][tid] = s_in[tid];
	}
	for (int k = tid; k < n; k += lm::BLOCK) a.level[e0 + k] = 0;
	__syncthreads();
	int cur = 0;
	int included = n;

	for (int rd = 0; rd < s.n; rd++) {
		const Round R = s.r[rd];
		if (R.restart && tid < 8) sh.state[cur][tid] = s_in[tid];
		__syncthreads();
		const Frame P = { a.edge, a.level, e0, n, nMono, s_cam, s.rk[rd] };
		const int nIt = lm::optimize(P, sh, included, R.iterations, a.stats ? a.stats + (size_t)b * s.statOff[s.n] + s.statOff[rd] : nullptr, cur);
		// ---- the outlier test on the committed pose (lv::k_classify_edges) ----
		int c4[4] = { 0, 0, 0, 0 };
		{
			double q[4], t[3], c[5];
			P.load(sh.state[cur], q, t, c);
			for (int k = tid; k < n; k += lm::BLOCK) {
				const bool stereo = k >= nMono;
				double X[3], m[3], om, Xc[3], r[3];
				load_edge(a.edge + 8 * (size_t)(e0 + k), X, m, om);
				if (!stereo) m[2] = 0;
				edge_residual(q, t, c, X, m, stereo, Xc, r);
				const double chi2 = om * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
				const bool fail = chi2 > R.chi2[stereo ? 1 : 0] || ((R.flags & lv::FAIL_DEPTH) && Xc[2] <= 0);
				const int old = a.level[e0 + k];
				const int now = (R.flags & lv::REINCLUDE) ? (fail ? 1 : 0) : (old | (fail ? 1 : 0));
				if (now != old) a.level[e0 + k] = (unsigned char)now;
				c4[0] += !now && !stereo; c4[1] += !now && stereo; c4[2] += !old && now; c4[3] += old && !now;
			}
		}
		// the barriers of block_count also order this round's reads of the state and levels before the next round's writes
#pragma unroll
		for (int k = 0; k < 4; k++) c4[k] = lm::block_count(c4[k], sh.cnt);
		included = c4[0] + c4[1];
		if (tid < 4) a.counts[((size_t)b * s.n + rd) * 4 + tid] = c4[tid];
		if (tid == 0) a.nstats[(size_t)b * s.n + rd] = nIt;
	}
	if (tid < 8) a.poseOut[8 * (size_t)b + tid] = tid < 7 ? sh.state[cur][tid] : 0.0;
}

}  // namespace pb
}  // namespace cuba_b200
