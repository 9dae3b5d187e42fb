// cuba_pose_batch.cuh -- pose optimisation of many frames in one launch (ORB-SLAM2's Optimizer::PoseOptimization, batched).
//
// A frame is one free SE(3) pose and its monocular / stereo edges, each with its own world point held fixed.  k_pose_batch runs one
// CTA per frame over the whole round schedule: per round an optional restart from the input pose, the LM loop of Engine::optimize
// (cuba_engine.cu) and the outlier test of lv::k_classify_edges on the committed pose.  Nothing leaves the CTA between rounds; the
// host reads the results once, after the launch.
//
// Per LM iteration a block-stride pass over the frame's edges at level 0 accumulates the 21 unique Hpp entries, bp and the robust
// chi2 (the formulas of k_linearize_pose); the damped 6x6 solve (spd6_inverse, as k_solve_poses_only) and the SE(3) update
// (se3_update) run in thread 0 and publish the trial pose in shared memory; every trial's chi2 pass reads it from there.  All sums
// are fixed-order warp trees followed by a fixed-order sum over the warps, so a frame's result is bit-reproducible and depends
// neither on the other frames of the batch nor on its position.  The sums over warps are done by every thread, which therefore
// holds the same F, lambda and nu and follows the same control flow without a broadcast.
//
// Edges are read from global memory on every pass (a frame of ~400 edges is 26 KB and stays in L1/L2); levels live in global
// memory, one byte per edge.
#pragma once

#include "cuba_kernels.cuh"

namespace cuba_b200 {
namespace pb {

constexpr int BLOCK = 128;            // threads per frame
constexpr int NW = BLOCK / 32;
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

// the layout of cuba_iter_stat
struct IterStat { int iteration, trials; double chi2, lambda; int pcg_iters, pcg_failed; };

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
	IterStat* stats;                  // [B][statOff[n]] or null
};

// fixed-order block sum whose result every thread receives (s_red: NW doubles)
__device__ __forceinline__ double block_sum_all(double v, double* s_red)
{
	v = warp_sum(v);
	if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
	__syncthreads();
	double r = 0;
#pragma unroll
	for (int i = 0; i < NW; i++) r += s_red[i];
	__syncthreads();
	return r;
}

__device__ __forceinline__ void load_edge(const double* __restrict__ p, double X[3], double m[3], double& om)
{
	ld2(p, X[0], X[1]); ld2(p + 2, X[2], m[0]); ld2(p + 4, m[1], m[2]);
	double pad;
	ld2(p + 6, om, pad);
}

// robust chi2 of the frame's included edges at the pose in shared memory
__device__ __forceinline__ double frame_chi2(const Args& a, int e0, int n, int nMono, const double* q, const double* t, const double* c,
	const RobustParams& rk, double* s_red)
{
	double chi = 0;
	for (int k = threadIdx.x; k < n; k += BLOCK) {
		if (a.level[e0 + k]) continue;
		const bool stereo = k >= nMono;
		double X[3], m[3], om, Xc[3], r[3], rho, drho;
		load_edge(a.edge + 8 * (size_t)(e0 + k), X, m, om);
		if (!stereo) m[2] = 0;
		edge_residual(q, t, c, X, m, stereo, Xc, r);
		const double e2 = om * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
		robust<double>(rk.type[stereo ? 1 : 0], rk.delta[stereo ? 1 : 0], e2, rho, drho);
		chi += rho;
	}
	return block_sum_all(chi, s_red);
}

__global__ void __launch_bounds__(BLOCK) k_pose_batch(const Args a, const Schedule s)
{
	__shared__ double s_part[NW][28];
	__shared__ double s_sys[28];          // 21 upper Hpp entries (column n, row l <= n at n (n+1)/2 + l), bp, chi2
	__shared__ double s_pose[2][8];       // committed / trial pose: q(4) t(3) pad
	__shared__ double s_in[8], s_cam[8];
	__shared__ double s_red[NW];
	__shared__ double s_scale;
	__shared__ int s_cnt[NW][4];

	const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	const int e0 = a.ptr2[b] + a.ptr3[b];
	const int nMono = a.ptr2[b + 1] - a.ptr2[b];
	const int n = nMono + a.ptr3[b + 1] - a.ptr3[b];
	if (tid < 8) {
		s_in[tid] = a.pose[8 * (size_t)b + tid];
		s_cam[tid] = a.cam[8 * (size_t)b + tid];
		s_pose[0][tid] = s_in[tid];
	}
	for (int k = tid; k < n; k += BLOCK) a.level[e0 + k] = 0;
	__syncthreads();
	int cur = 0;
	int included = n;

	for (int rd = 0; rd < s.n; rd++) {
		const Round R = s.r[rd];
		const RobustParams rk = s.rk[rd];
		if (R.restart && tid < 8) s_pose[cur][tid] = s_in[tid];
		__syncthreads();
		int nIt = 0;
		// ---- the LM loop of Engine::optimize; a round without an included edge writes no iteration and leaves the pose alone ----
		if (included > 0) {
			const double tau = 1e-5;
			double nu = 2, lambda = 0, F = 0;
			for (int it = 0; it < R.iterations; it++) {
				// linearise at the committed pose
				double acc[28];
#pragma unroll
				for (int i = 0; i < 28; i++) acc[i] = 0;
				{
					double q[4], t[3], c[5];
#pragma unroll
					for (int i = 0; i < 4; i++) q[i] = s_pose[cur][i];
#pragma unroll
					for (int i = 0; i < 3; i++) t[i] = s_pose[cur][4 + i];
#pragma unroll
					for (int i = 0; i < 5; i++) c[i] = s_cam[i];
					for (int k = tid; k < n; k += BLOCK) {
						if (a.level[e0 + k]) continue;
						const bool stereo = k >= nMono;
						double X[3], m[3], om, Xc[3], r[3], rho, drho;
						load_edge(a.edge + 8 * (size_t)(e0 + k), X, m, om);
						if (!stereo) m[2] = 0;
						edge_residual(q, t, c, X, m, stereo, Xc, r);
						const double e2 = om * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
						robust<double>(rk.type[stereo ? 1 : 0], rk.delta[stereo ? 1 : 0], e2, rho, drho);
						acc[27] += rho;
						const double w = om * drho;
						double JP[3][6], JL[3][3], wJP[3][6];
						edge_jacobians(q, c, Xc, stereo, JP, JL);
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
#pragma unroll
				for (int i = 0; i < 28; i++) {
					const double v = warp_sum(acc[i]);
					if (lane == 0) s_part[wid][i] = v;
				}
				__syncthreads();
				if (tid < 28) {
					double v = 0;
#pragma unroll
					for (int w = 0; w < NW; w++) v += s_part[w][tid];
					s_sys[tid] = v;
				}
				__syncthreads();
				F = s_sys[27];
				if (it == 0) {
					double md = 0;     // k_max_diagonal: the largest diagonal entry, starting from 0
#pragma unroll
					for (int d = 0; d < 6; d++) { const double v = s_sys[d * (d + 1) / 2 + d]; md = v > md ? v : md; }
					lambda = tau * md;
				}
				int q = 0, trials = 0;
				double rho = -1;
				for (; q < 10 && rho < 0; q++) {
					trials++;
					// damped solve and SE(3) update of the trial pose (k_solve_poses_only + k_update_poses)
					if (tid == 0) {
						double M[36], xp[6];
						for (int e = 0; e < 36; e++) {
							const int cn = e / 6, l = e - 6 * cn;
							const int lo = l < cn ? l : cn, hi = l < cn ? cn : l;
							M[e] = s_sys[hi * (hi + 1) / 2 + lo] + ((e % 7) == 0 ? lambda : 0.0);
						}
						if (!spd6_inverse(M)) {
							for (int i = 0; i < 6; i++) xp[i] = 0;
						} else {
							for (int r = 0; r < 6; r++) {
								double sum = 0;
								for (int c = 0; c < 6; c++) sum += M[c * 6 + r] * s_sys[21 + c];
								xp[r] = sum;
							}
						}
						double qq[4], tt[3];
						for (int i = 0; i < 4; i++) qq[i] = s_pose[cur][i];
						for (int i = 0; i < 3; i++) tt[i] = s_pose[cur][4 + i];
						se3_update(xp, qq, tt);
						for (int i = 0; i < 4; i++) s_pose[cur ^ 1][i] = qq[i];
						for (int i = 0; i < 3; i++) s_pose[cur ^ 1][4 + i] = tt[i];
						double sc = 0;
						for (int i = 0; i < 6; i++) sc += xp[i] * (lambda * xp[i] + s_sys[21 + i]);
						s_scale = sc;
					}
					__syncthreads();
					const double scale = s_scale + 1e-3;   // read before the pass: thread 0 rewrites it once the pass's barriers are behind it
					double Fhat;
					{
						double qt[4], tt[3], c[5];
#pragma unroll
						for (int i = 0; i < 4; i++) qt[i] = s_pose[cur ^ 1][i];
#pragma unroll
						for (int i = 0; i < 3; i++) tt[i] = s_pose[cur ^ 1][4 + i];
#pragma unroll
						for (int i = 0; i < 5; i++) c[i] = s_cam[i];
						Fhat = frame_chi2(a, e0, n, nMono, qt, tt, c, rk, s_red);
					}
					rho = (F - Fhat) / scale;
					if (!(rho == rho)) rho = -1;   // NaN trial -> reject
					if (rho > 0) {
						const double x = 2 * rho - 1;
						lambda *= fmax(1. / 3, fmin(1 - x * x * x, 2. / 3));
						nu = 2; F = Fhat;
						cur ^= 1;
						break;
					} else {
						lambda *= nu; nu *= 2;
					}
				}
				if (tid == 0 && a.stats) {
					IterStat& st = a.stats[(size_t)b * s.statOff[s.n] + s.statOff[rd] + nIt];
					st.iteration = it; st.trials = trials; st.chi2 = F; st.lambda = lambda; st.pcg_iters = 0; st.pcg_failed = 0;
				}
				nIt++;
				__syncthreads();     // s_sys and the trial buffer are rewritten by the next iteration
				if (q == 10 || rho <= 0 || !isfinite(lambda)) break;
			}
		}
		// ---- the outlier test on the committed pose (lv::k_classify_edges) ----
		int c4[4] = { 0, 0, 0, 0 };
		{
			double q[4], t[3], c[5];
#pragma unroll
			for (int i = 0; i < 4; i++) q[i] = s_pose[cur][i];
#pragma unroll
			for (int i = 0; i < 3; i++) t[i] = s_pose[cur][4 + i];
#pragma unroll
			for (int i = 0; i < 5; i++) c[i] = s_cam[i];
			for (int k = tid; k < n; k += BLOCK) {
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
#pragma unroll
		for (int k = 0; k < 4; k++) {
			int v = c4[k];
#pragma unroll
			for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
			if (lane == 0) s_cnt[wid][k] = v;
		}
		__syncthreads();
#pragma unroll
		for (int k = 0; k < 4; k++) {
			int v = 0;
#pragma unroll
			for (int w = 0; w < NW; w++) v += s_cnt[w][k];
			c4[k] = v;
		}
		included = c4[0] + c4[1];
		if (tid < 4) a.counts[((size_t)b * s.n + rd) * 4 + tid] = c4[tid];
		if (tid == 0) a.nstats[(size_t)b * s.n + rd] = nIt;
		__syncthreads();     // s_cnt and the levels are read again by the next round
	}
	if (tid < 8) a.poseOut[8 * (size_t)b + tid] = tid < 7 ? s_pose[cur][tid] : 0.0;
}

}  // namespace pb
}  // namespace cuba_b200
