// cuba_sim3_batch.cuh -- Sim(3) alignment of many keyframe pairs in one launch (ORB-SLAM2's Optimizer::OptimizeSim3, batched).
//
// A problem is keyframes 1 and 2 and N matched pairs; pair i carries X1 (camera-1 coordinates), X2 (camera-2 coordinates), the
// keypoints obs1 / obs2 and scalar informations omega1 / omega2.  The unknown is S12 = (R(q), t, s), S X = s R X + t.  Each pair
// gives two monocular edges under a Huber kernel with delta = sqrt(chi2):
//   e12: r = pi1(S12 X2) - obs1          e21: r = pi2(S12^-1 X1) - obs2
// The update is S <- Exp(xi) S, xi = (omega, upsilon, sigma) (sim3_update of cuba_math.cuh, with its residuals and analytic
// Jacobians); with fix_scale the sigma column of every Jacobian is zero, so the damped solve gives sigma = 0 and s stays bit for bit.
//
// k_sim3_batch runs one CTA per problem over OptimizeSim3's whole schedule:
//   1. optimize(iterations) over every pair, under the LM rules of Engine::optimize (lm_* below, as k_pose_batch);
//   2. the pair test on the committed S: a pair fails when either edge's omega |r|^2 exceeds chi2; failed pairs go to level 1;
//   3. fewer than min_pairs pairs left: 0 inliers and S is the input S.  Otherwise optimize(n) over the pairs left, n =
//      iterations_bad if step 2 removed a pair, else iterations_good;
//   4. the same test again; the pairs still at level 0 are the inliers.
// Per LM iteration a block-stride pass over the problem's pairs at level 0 accumulates the 28 upper H entries, b (7) and the robust
// chi2; thread 0 solves the damped 7x7 system (spd_inverse<7>), applies the update and publishes the trial S in shared memory.  All
// sums are fixed-order warp trees followed by a fixed-order sum over the warps done by every thread, so a problem's result is
// bit-reproducible and depends neither on the other problems of the batch nor on its position.  Pairs are read from global memory
// on every pass; levels live in global memory, one byte per pair.
#pragma once

#include "cuba_pose_batch.cuh"

namespace cuba_b200 {
namespace s3 {

constexpr int BLOCK = pb::BLOCK;      // threads per problem
constexpr int NW = BLOCK / 32;
constexpr int PROB = 20;              // doubles per problem record: q(4) t(3) s cam1(4) cam2(4) fix_scale pad(3)
constexpr int PAIR = 12;              // doubles per pair record: X1(3) X2(3) obs1(2) obs2(2) omega1 omega2
constexpr int NSYS = 28 + 7 + 1;      // H (upper, packed as lm_*), b, chi2

struct Args {
	int B;
	const double* prob;               // [B][PROB]
	const double* pair;               // [N][PAIR]; problem b: ptr[b] .. ptr[b+1]
	const int* ptr;                   // [B+1]
	double* Sout;                     // [B][8]  q(4) t(3) s
	unsigned char* level;             // [N]
	int* ninliers;                    // [B]
	int* nstats;                      // [B][2]
	pb::IterStat* stats;              // [B][statPer] or null
};
struct Params {
	double chi2, delta;
	int iterations, iterationsBad, iterationsGood, minPairs;
	int statPer;                      // stat slots per problem: iterations + max(iterationsBad, iterationsGood)
};

// ---- the LM control of Engine::optimize, restated from k_pose_batch for N unknowns.  (Calling these helpers from k_pose_batch
// changes its register allocation, so k_pose_batch keeps its own copy of the loop and its SASS stays that of the kernel that was
// measured.)  The system is packed as sys[0 .. N(N+1)/2): the upper triangle (column n, row l <= n at n (n+1)/2 + l), then b =
// sys[N(N+1)/2 ..]; the step x solves (H + lambda I) x = b.
constexpr int LM_MAX_TRIALS = 10;

// lambda of the first iteration: tau times the largest diagonal entry, starting from 0 (k_max_diagonal)
template <int N>
__device__ __forceinline__ double lm_initial_lambda(const double* sys)
{
	const double tau = 1e-5;
	double md = 0;
#pragma unroll
	for (int d = 0; d < N; d++) { const double v = sys[d * (d + 1) / 2 + d]; md = v > md ? v : md; }
	return tau * md;
}

// the damped solve (k_solve_poses_only): x = 0 when the Cholesky of H + lambda I fails
template <int N>
__device__ __forceinline__ void lm_damped_solve(const double* sys, double lambda, double x[N])
{
	double M[N * N];
	for (int e = 0; e < N * N; e++) {
		const int cn = e / N, l = e - N * cn;
		const int lo = l < cn ? l : cn, hi = l < cn ? cn : l;
		M[e] = sys[hi * (hi + 1) / 2 + lo] + ((e % (N + 1)) == 0 ? lambda : 0.0);
	}
	if (!spd_inverse<N>(M)) {
		for (int i = 0; i < N; i++) x[i] = 0;
	} else {
		for (int r = 0; r < N; r++) {
			double sum = 0;
			for (int c = 0; c < N; c++) sum += M[c * N + r] * sys[N * (N + 1) / 2 + c];
			x[r] = sum;
		}
	}
}

// the predicted decrease x^T (lambda x + b), without the 1e-3 the gain ratio adds
template <int N>
__device__ __forceinline__ double lm_scale(const double* sys, double lambda, const double x[N])
{
	double sc = 0;
	for (int i = 0; i < N; i++) sc += x[i] * (lambda * x[i] + sys[N * (N + 1) / 2 + i]);
	return sc;
}

// the gain ratio rho of a trial (a NaN trial is rejected) and the lambda / nu update it implies; an accepted trial's chi2 becomes F.
// Returns whether the trial was accepted.
__device__ __forceinline__ bool lm_trial(double& F, double Fhat, double scale, double& lambda, double& nu, double& rho)
{
	rho = (F - Fhat) / scale;
	if (!(rho == rho)) rho = -1;
	if (rho > 0) {
		const double x = 2 * rho - 1;
		lambda *= fmax(1. / 3, fmin(1 - x * x * x, 2. / 3));
		nu = 2; F = Fhat;
		return true;
	}
	lambda *= nu; nu *= 2;
	return false;
}

// the end of the iterations: every trial rejected, no decrease, or lambda no longer finite
__device__ __forceinline__ bool lm_stop(int trials, double rho, double lambda)
{
	return trials == LM_MAX_TRIALS || rho <= 0 || !isfinite(lambda);
}

__device__ __forceinline__ void load_pair(const double* __restrict__ p, double X1[3], double X2[3], double o1[2], double o2[2], double& om1, double& om2)
{
	ld2(p, X1[0], X1[1]); ld2(p + 2, X1[2], X2[0]); ld2(p + 4, X2[1], X2[2]);
	ld2(p + 6, o1[0], o1[1]); ld2(p + 8, o2[0], o2[1]); ld2(p + 10, om1, om2);
}

// fixed-order block sum of an int whose result every thread receives (s_cnt: NW ints)
__device__ __forceinline__ int block_count(int v, int* s_cnt)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	if ((threadIdx.x & 31) == 0) s_cnt[threadIdx.x >> 5] = v;
	__syncthreads();
	int r = 0;
#pragma unroll
	for (int i = 0; i < NW; i++) r += s_cnt[i];
	__syncthreads();
	return r;
}

// robust chi2 of the problem's pairs at level 0 at S = (q, t, s)
__device__ __forceinline__ double problem_chi2(const Args& a, int i0, int n, const double* S, const double* c1, const double* c2, double delta,
	double* s_red)
{
	double chi = 0;
	for (int k = threadIdx.x; k < n; k += BLOCK) {
		if (a.level[i0 + k]) continue;
		double X1[3], X2[3], o1[2], o2[2], om1, om2, P[3], r[2], rho, drho;
		load_pair(a.pair + PAIR * (size_t)(i0 + k), X1, X2, o1, o2, om1, om2);
		sim3_residual12(S, S + 4, S[7], c1, X2, o1, P, r);
		robust<double>(RK_HUBER, delta, om1 * (r[0] * r[0] + r[1] * r[1]), rho, drho);
		chi += rho;
		sim3_residual21(S, S + 4, S[7], c2, X1, o2, P, r);
		robust<double>(RK_HUBER, delta, om2 * (r[0] * r[0] + r[1] * r[1]), rho, drho);
		chi += rho;
	}
	return pb::block_sum_all(chi, s_red);
}

// H += w J^T J (upper, packed), b -= w J^T r for one edge
__device__ __forceinline__ void accumulate(double acc[NSYS], const double J[2][7], const double r[2], double w)
{
	double wJ[2][7];
#pragma unroll
	for (int m = 0; m < 2; m++)
#pragma unroll
		for (int l = 0; l < 7; l++) wJ[m][l] = w * J[m][l];
	int kk = 0;
#pragma unroll
	for (int cn = 0; cn < 7; cn++)
#pragma unroll
		for (int l = 0; l <= cn; l++) {
			acc[kk] += J[0][l] * wJ[0][cn] + J[1][l] * wJ[1][cn];
			kk++;
		}
#pragma unroll
	for (int l = 0; l < 7; l++) acc[28 + l] -= wJ[0][l] * r[0] + wJ[1][l] * r[1];
}

struct Shared {
	double part[NW][NSYS];
	double sys[NSYS];
	double S[2][8];                   // committed / trial S: q(4) t(3) s
	double cam[8];                    // cam1(4) cam2(4)
	double red[NW];
	double scale;
	int cnt[NW];
};

// optimize(iterations) over the pairs at level 0 from S[cur] (the LM loop of Engine::optimize); writes the iteration statistics
// from slot statBase and returns the number written.  No pair at level 0: no iteration, S alone.
__device__ __forceinline__ int optimize(const Args& a, const Params& p, Shared& sh, int b, int i0, int n, int included, int iterations,
	int statBase, bool fixScale, int& cur)
{
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	if (included == 0) return 0;
	int nIt = 0;
	double nu = 2, lambda = 0, F = 0;
	for (int it = 0; it < iterations; it++) {
		// linearise at the committed S
		double acc[NSYS];
#pragma unroll
		for (int i = 0; i < NSYS; i++) acc[i] = 0;
		{
			double S[8], c1[4], c2[4];
#pragma unroll
			for (int i = 0; i < 8; i++) S[i] = sh.S[cur][i];
#pragma unroll
			for (int i = 0; i < 4; i++) { c1[i] = sh.cam[i]; c2[i] = sh.cam[4 + i]; }
			for (int k = tid; k < n; k += BLOCK) {
				if (a.level[i0 + k]) continue;
				double X1[3], X2[3], o1[2], o2[2], om1, om2, P[3], r[2], J[2][7], rho, drho;
				load_pair(a.pair + PAIR * (size_t)(i0 + k), X1, X2, o1, o2, om1, om2);
				// e12
				sim3_residual12(S, S + 4, S[7], c1, X2, o1, P, r);
				robust<double>(RK_HUBER, p.delta, om1 * (r[0] * r[0] + r[1] * r[1]), rho, drho);
				acc[NSYS - 1] += rho;
				sim3_jacobian12(c1, P, J);
				if (fixScale) J[0][6] = J[1][6] = 0;
				accumulate(acc, J, r, om1 * drho);
				// e21
				sim3_residual21(S, S + 4, S[7], c2, X1, o2, P, r);
				robust<double>(RK_HUBER, p.delta, om2 * (r[0] * r[0] + r[1] * r[1]), rho, drho);
				acc[NSYS - 1] += rho;
				sim3_jacobian21(S, S[7], c2, X1, P, J);
				if (fixScale) J[0][6] = J[1][6] = 0;
				accumulate(acc, J, r, om2 * drho);
			}
		}
#pragma unroll
		for (int i = 0; i < NSYS; i++) {
			const double v = warp_sum(acc[i]);
			if (lane == 0) sh.part[wid][i] = v;
		}
		__syncthreads();
		if (tid < NSYS) {
			double v = 0;
#pragma unroll
			for (int w = 0; w < NW; w++) v += sh.part[w][tid];
			sh.sys[tid] = v;
		}
		__syncthreads();
		F = sh.sys[NSYS - 1];
		if (it == 0) lambda = lm_initial_lambda<7>(sh.sys);
		int q = 0, trials = 0;
		double rho = -1;
		for (; q < LM_MAX_TRIALS && rho < 0; q++) {
			trials++;
			// damped solve and Sim(3) update of the trial S
			if (tid == 0) {
				double x[7];
				lm_damped_solve<7>(sh.sys, lambda, x);
				double qq[4], tt[3], ss = sh.S[cur][7];
				for (int i = 0; i < 4; i++) qq[i] = sh.S[cur][i];
				for (int i = 0; i < 3; i++) tt[i] = sh.S[cur][4 + i];
				sim3_update(x, qq, tt, ss);
				for (int i = 0; i < 4; i++) sh.S[cur ^ 1][i] = qq[i];
				for (int i = 0; i < 3; i++) sh.S[cur ^ 1][4 + i] = tt[i];
				sh.S[cur ^ 1][7] = ss;
				sh.scale = lm_scale<7>(sh.sys, lambda, x);
			}
			__syncthreads();
			const double scale = sh.scale + 1e-3;   // read before the pass: thread 0 rewrites it once the pass's barriers are behind it
			double Fhat;
			{
				double S[8], c1[4], c2[4];
#pragma unroll
				for (int i = 0; i < 8; i++) S[i] = sh.S[cur ^ 1][i];
#pragma unroll
				for (int i = 0; i < 4; i++) { c1[i] = sh.cam[i]; c2[i] = sh.cam[4 + i]; }
				Fhat = problem_chi2(a, i0, n, S, c1, c2, p.delta, sh.red);
			}
			if (lm_trial(F, Fhat, scale, lambda, nu, rho)) {
				cur ^= 1;
				break;
			}
		}
		if (tid == 0 && a.stats) {
			pb::IterStat& st = a.stats[(size_t)b * p.statPer + statBase + nIt];
			st.iteration = it; st.trials = trials; st.chi2 = F; st.lambda = lambda; st.pcg_iters = 0; st.pcg_failed = 0;
		}
		nIt++;
		__syncthreads();     // sys and the trial S are rewritten by the next iteration
		if (lm_stop(q, rho, lambda)) break;
	}
	return nIt;
}

// the pair test on S[cur] over the pairs at level 0: a failing pair goes to level 1.  Returns (pairs left at level 0, pairs removed).
__device__ __forceinline__ void test_pairs(const Args& a, const Params& p, Shared& sh, int i0, int n, int cur, int& left, int& removed)
{
	double S[8], c1[4], c2[4];
#pragma unroll
	for (int i = 0; i < 8; i++) S[i] = sh.S[cur][i];
#pragma unroll
	for (int i = 0; i < 4; i++) { c1[i] = sh.cam[i]; c2[i] = sh.cam[4 + i]; }
	int nLeft = 0, nRem = 0;
	for (int k = threadIdx.x; k < n; k += BLOCK) {
		if (a.level[i0 + k]) continue;
		double X1[3], X2[3], o1[2], o2[2], om1, om2, P[3], r[2];
		load_pair(a.pair + PAIR * (size_t)(i0 + k), X1, X2, o1, o2, om1, om2);
		sim3_residual12(S, S + 4, S[7], c1, X2, o1, P, r);
		const double e12 = om1 * (r[0] * r[0] + r[1] * r[1]);
		sim3_residual21(S, S + 4, S[7], c2, X1, o2, P, r);
		const double e21 = om2 * (r[0] * r[0] + r[1] * r[1]);
		if (e12 > p.chi2 || e21 > p.chi2) { a.level[i0 + k] = 1; nRem++; }
		else nLeft++;
	}
	left = block_count(nLeft, sh.cnt);
	removed = block_count(nRem, sh.cnt);
}

__global__ void __launch_bounds__(BLOCK) k_sim3_batch(const Args a, const Params p)
{
	__shared__ Shared sh;
	const int b = blockIdx.x, tid = threadIdx.x;
	const int i0 = a.ptr[b], n = a.ptr[b + 1] - i0;
	const double* P = a.prob + PROB * (size_t)b;
	if (tid < 8) {
		sh.S[0][tid] = P[tid];
		sh.cam[tid] = P[8 + tid];
	}
	const bool fixScale = P[16] != 0;
	for (int k = tid; k < n; k += BLOCK) a.level[i0 + k] = 0;
	__syncthreads();
	int cur = 0;
	// 1. optimize(iterations) over every pair, 2. the pair test
	const int n0 = optimize(a, p, sh, b, i0, n, n, p.iterations, 0, fixScale, cur);
	int left, removed;
	test_pairs(a, p, sh, i0, n, cur, left, removed);
	int n1 = 0, inliers = 0;
	if (left >= p.minPairs) {
		// 3. optimize(iterations_bad or iterations_good) over the pairs left, 4. the test again
		n1 = optimize(a, p, sh, b, i0, n, left, removed > 0 ? p.iterationsBad : p.iterationsGood, p.iterations, fixScale, cur);
		int removed2;
		test_pairs(a, p, sh, i0, n, cur, inliers, removed2);
	}
	if (tid < 8) a.Sout[8 * (size_t)b + tid] = left >= p.minPairs ? sh.S[cur][tid] : P[tid];
	if (tid == 0) {
		a.ninliers[b] = inliers;
		a.nstats[2 * (size_t)b] = n0;
		a.nstats[2 * (size_t)b + 1] = n1;
	}
}

}  // namespace s3
}  // namespace cuba_b200
