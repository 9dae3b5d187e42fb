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
//   1. optimize(iterations) over every pair: the LM loop of Engine::optimize (lm::optimize, cuba_lm_batch.cuh);
//   2. the pair test on the committed S: a pair fails when either edge's omega |r|^2 exceeds chi2; failed pairs go to level 1;
//   3. fewer than min_pairs pairs left: 0 inliers and S is the input S.  Otherwise optimize(n) over the pairs left, n =
//      iterations_bad if step 2 removed a pair, else iterations_good;
//   4. the same test again; the pairs still at level 0 are the inliers.
// Per LM iteration a block-stride pass over the problem's pairs at level 0 accumulates the 28 upper H entries, b (7) and the robust
// chi2; the damped 7x7 solve is spd_inverse<7> and the update sim3_update.  Pairs are read from global memory on every pass; levels
// live in global memory, one byte per pair.
#pragma once

#include "cuba_lm_batch.cuh"

namespace cuba_b200 {
namespace s3 {

constexpr int PROB = 20;              // doubles per problem record: q(4) t(3) s cam1(4) cam2(4) fix_scale pad(3)
constexpr int PAIR = 12;              // doubles per pair record: X1(3) X2(3) obs1(2) obs2(2) omega1 omega2

struct Args {
	int B;
	const double* prob;               // [B][PROB]
	const double* pair;               // [N][PAIR]; problem b: ptr[b] .. ptr[b+1]
	const int* ptr;                   // [B+1]
	double* Sout;                     // [B][8]  q(4) t(3) s
	unsigned char* level;             // [N]
	int* ninliers;                    // [B]
	int* nstats;                      // [B][2]
	lm::IterStat* stats;              // [B][statPer] or null
};
struct Params {
	double chi2, delta;
	int iterations, iterationsBad, iterationsGood, minPairs;
	int statPer;                      // stat slots per problem: iterations + max(iterationsBad, iterationsGood)
};

__device__ __forceinline__ void load_pair(const double* __restrict__ p, double X1[3], double X2[3], double o1[2], double o2[2], double& om1, double& om2)
{
	ld2(p, X1[0], X1[1]); ld2(p + 2, X1[2], X2[0]); ld2(p + 4, X2[1], X2[2]);
	ld2(p + 6, o1[0], o1[1]); ld2(p + 8, o2[0], o2[1]); ld2(p + 10, om1, om2);
}

// H += w J^T J (upper, packed), b -= w J^T r for one edge
__device__ __forceinline__ void accumulate(double acc[36], const double J[2][7], const double r[2], double w)
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

// one problem's LM problem over its pairs at level 0; the state is S = q(4) t(3) s
struct Problem {
	static constexpr int N = 7;
	const double* pair;               // the problem's pairs
	unsigned char* level;
	int n;
	const double* cam;                // cam1(4) cam2(4), shared memory
	double delta;
	bool fixScale;

	__device__ __forceinline__ void load(const double* Sh, double S[8], double c1[4], double c2[4]) const
	{
#pragma unroll
		for (int i = 0; i < 8; i++) S[i] = Sh[i];
#pragma unroll
		for (int i = 0; i < 4; i++) { c1[i] = cam[i]; c2[i] = cam[4 + i]; }
	}

	__device__ __forceinline__ void linearize(double acc[36], const double* Sh) const
	{
		double S[8], c1[4], c2[4];
		load(Sh, S, c1, c2);
		for (int k = threadIdx.x; k < n; k += lm::BLOCK) {
			if (level[k]) continue;
			double X1[3], X2[3], o1[2], o2[2], om1, om2, P[3], r[2], J[2][7], rho, drho;
			load_pair(pair + PAIR * (size_t)k, X1, X2, o1, o2, om1, om2);
			// e12
			sim3_residual12(S, S + 4, S[7], c1, X2, o1, P, r);
			robust<double>(RK_HUBER, delta, om1 * (r[0] * r[0] + r[1] * r[1]), rho, drho);
			acc[35] += rho;
			sim3_jacobian12(c1, P, J);
			if (fixScale) J[0][6] = J[1][6] = 0;
			accumulate(acc, J, r, om1 * drho);
			// e21
			sim3_residual21(S, S + 4, S[7], c2, X1, o2, P, r);
			robust<double>(RK_HUBER, delta, om2 * (r[0] * r[0] + r[1] * r[1]), rho, drho);
			acc[35] += rho;
			sim3_jacobian21(S, S[7], c2, X1, P, J);
			if (fixScale) J[0][6] = J[1][6] = 0;
			accumulate(acc, J, r, om2 * drho);
		}
	}

	__device__ __forceinline__ double chi2(const double* Sh) const
	{
		double S[8], c1[4], c2[4];
		load(Sh, S, c1, c2);
		double chi = 0;
		for (int k = threadIdx.x; k < n; k += lm::BLOCK) {
			if (level[k]) continue;
			double X1[3], X2[3], o1[2], o2[2], om1, om2, P[3], r[2], rho, drho;
			load_pair(pair + PAIR * (size_t)k, X1, X2, o1, o2, om1, om2);
			sim3_residual12(S, S + 4, S[7], c1, X2, o1, P, r);
			robust<double>(RK_HUBER, delta, om1 * (r[0] * r[0] + r[1] * r[1]), rho, drho);
			chi += rho;
			sim3_residual21(S, S + 4, S[7], c2, X1, o2, P, r);
			robust<double>(RK_HUBER, delta, om2 * (r[0] * r[0] + r[1] * r[1]), rho, drho);
			chi += rho;
		}
		return chi;
	}

	__device__ __forceinline__ void update(const double x[7], const double* S, double* St) const
	{
		double qq[4], tt[3], ss = S[7];
		for (int i = 0; i < 4; i++) qq[i] = S[i];
		for (int i = 0; i < 3; i++) tt[i] = S[4 + i];
		sim3_update(x, qq, tt, ss);
		for (int i = 0; i < 4; i++) St[i] = qq[i];
		for (int i = 0; i < 3; i++) St[4 + i] = tt[i];
		St[7] = ss;
	}

	// the pair test at S over the pairs at level 0: a failing pair goes to level 1.  Returns (pairs left at level 0, pairs removed).
	__device__ __forceinline__ void test(const double* Sh, double chi2, int* s_cnt, int& left, int& removed) const
	{
		double S[8], c1[4], c2[4];
		load(Sh, S, c1, c2);
		int nLeft = 0, nRem = 0;
		for (int k = threadIdx.x; k < n; k += lm::BLOCK) {
			if (level[k]) continue;
			double X1[3], X2[3], o1[2], o2[2], om1, om2, P[3], r[2];
			load_pair(pair + PAIR * (size_t)k, X1, X2, o1, o2, om1, om2);
			sim3_residual12(S, S + 4, S[7], c1, X2, o1, P, r);
			const double e12 = om1 * (r[0] * r[0] + r[1] * r[1]);
			sim3_residual21(S, S + 4, S[7], c2, X1, o2, P, r);
			const double e21 = om2 * (r[0] * r[0] + r[1] * r[1]);
			if (e12 > chi2 || e21 > chi2) { level[k] = 1; nRem++; }
			else nLeft++;
		}
		left = lm::block_count(nLeft, s_cnt);
		removed = lm::block_count(nRem, s_cnt);
	}
};

__global__ void __launch_bounds__(lm::BLOCK) k_sim3_batch(const Args a, const Params p)
{
	__shared__ lm::Shared<Problem::N> sh;
	__shared__ double s_cam[8];
	const int b = blockIdx.x, tid = threadIdx.x;
	const int i0 = a.ptr[b], n = a.ptr[b + 1] - i0;
	const double* P = a.prob + PROB * (size_t)b;
	if (tid < 8) {
		sh.state[0][tid] = P[tid];
		s_cam[tid] = P[8 + tid];
	}
	const Problem pr = { a.pair + PAIR * (size_t)i0, a.level + i0, n, s_cam, p.delta, P[16] != 0 };
	for (int k = tid; k < n; k += lm::BLOCK) a.level[i0 + k] = 0;
	__syncthreads();
	lm::IterStat* stats = a.stats ? a.stats + (size_t)b * p.statPer : nullptr;
	int cur = 0;
	// 1. optimize(iterations) over every pair, 2. the pair test
	const int n0 = lm::optimize(pr, sh, n, p.iterations, stats, cur);
	int left, removed;
	pr.test(sh.state[cur], p.chi2, sh.cnt, left, removed);
	int n1 = 0, inliers = 0;
	if (left >= p.minPairs) {
		// 3. optimize(iterations_bad or iterations_good) over the pairs left, 4. the test again
		n1 = lm::optimize(pr, sh, left, removed > 0 ? p.iterationsBad : p.iterationsGood, stats ? stats + p.iterations : nullptr, cur);
		int removed2;
		pr.test(sh.state[cur], p.chi2, sh.cnt, inliers, removed2);
	}
	if (tid < 8) a.Sout[8 * (size_t)b + tid] = left >= p.minPairs ? sh.state[cur][tid] : P[tid];
	if (tid == 0) {
		a.ninliers[b] = inliers;
		a.nstats[2 * (size_t)b] = n0;
		a.nstats[2 * (size_t)b + 1] = n1;
	}
}

}  // namespace s3
}  // namespace cuba_b200
