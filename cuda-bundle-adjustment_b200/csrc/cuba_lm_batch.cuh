// cuba_lm_batch.cuh -- the block-level LM loop of the batched kernels (k_pose_batch, k_sim3_batch): one CTA of BLOCK threads runs
// Engine::optimize's LM loop (the rules in lm:: of cuba_math.cuh) on one small problem of N unknowns.
//
// Per iteration every thread accumulates its share of the packed system at the committed state; thread 0 solves the damped system,
// applies the update and publishes the trial state and its predicted decrease in shared memory; every trial's chi2 pass reads the
// trial state from there.  All sums are fixed-order warp trees followed by a fixed-order sum over the warps, so a problem's result is
// bit-reproducible and depends neither on the other problems of the batch nor on its position.  The sums over warps are done by every
// thread, which therefore holds the same F, lambda and nu and follows the same control flow without a broadcast.
//
// optimize_warp is the same loop for one small problem per warp (k_point_batch), for problems of a few items each.
#pragma once

#include "cuba_kernels.cuh"

namespace cuba_b200 {
namespace lm {

constexpr int BLOCK = 128;            // threads per problem
constexpr int NW = BLOCK / 32;

// the layout of cuba_iter_stat
struct IterStat { int iteration, trials; double chi2, lambda; int pcg_iters, pcg_failed; };

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

// block sum of an int whose result every thread receives (s_cnt: NW ints)
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

template <int N>
struct Shared {
	static constexpr int NSYS = N * (N + 1) / 2 + N + 1;   // the packed system of cuba_math.cuh, then chi2
	double part[NW][NSYS];
	double sys[NSYS];
	double state[2][8];               // committed / trial state, in the problem's layout
	double red[NW];
	double predicted;
	int cnt[NW];
};

// optimize(iterations) from sh.state[cur]; an accepted trial flips cur.  The problem type supplies
//   N                   the number of unknowns
//   linearize(acc, S)   per thread: adds its items' share of the packed system and of the robust chi2 at state S to acc[NSYS]
//   chi2(S)             per thread: its items' robust chi2 at state S
//   update(x, S, St)    thread 0: St = S moved by the step x
// Writes one IterStat per iteration to stats[0 ..] unless stats is null and returns the number written.  With no item included: no
// iteration, the state alone.
template <class Problem>
__device__ __forceinline__ int optimize(const Problem& P, Shared<Problem::N>& sh, int included, int iterations, IterStat* stats, int& cur)
{
	constexpr int N = Problem::N, NSYS = Shared<N>::NSYS;
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	if (included == 0) return 0;
	double nu = 2, lambda = 0, F = 0;
	for (int it = 0; it < iterations; it++) {
		double acc[NSYS];
#pragma unroll
		for (int i = 0; i < NSYS; i++) acc[i] = 0;
		P.linearize(acc, sh.state[cur]);
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
		if (it == 0) lambda = initial_lambda(max_diagonal<N>(sh.sys));
		int q = 0, trials = 0;
		double rho = -1;
		for (; q < MAX_TRIALS && rho < 0; q++) {
			trials++;
			if (tid == 0) {
				double x[N];
				damped_solve<N>(sh.sys, lambda, x);
				P.update(x, sh.state[cur], sh.state[cur ^ 1]);
				sh.predicted = predicted_decrease<N>(sh.sys, lambda, x);
			}
			__syncthreads();
			const double predicted = sh.predicted;   // read before the pass: thread 0 rewrites it once the pass's barriers are behind it
			const double Fhat = block_sum_all(P.chi2(sh.state[cur ^ 1]), sh.red);
			rho = gain_ratio(F, Fhat, predicted);
			if (update_damping(rho, lambda, nu)) {
				F = Fhat;
				cur ^= 1;
				break;
			}
		}
		if (tid == 0 && stats) {
			IterStat& st = stats[it];
			st.iteration = it; st.trials = trials; st.chi2 = F; st.lambda = lambda; st.pcg_iters = 0; st.pcg_failed = 0;
		}
		__syncthreads();     // sys and the trial state are rewritten by the next iteration
		if (stop(q, rho, lambda)) return it + 1;
	}
	return iterations;
}

// optimize(iterations) of one problem per WARP (k_point_batch): the loop of optimize above with the state X[N] in registers.  Every
// entry of the packed system and every chi2 is a warp_sum, whose xor butterfly leaves bitwise the same value in every lane, so every
// lane solves, updates and decides identically: no shared memory, no broadcast, no barrier.  The problem type supplies
//   N                   the number of unknowns, and the size of the state
//   linearize(acc, X)   per lane: adds its items' share of the packed system and of the robust chi2 at state X to acc[NSYS]
//   chi2(X)             per lane: its items' robust chi2 at state X
//   solve(sys, lambda, x)   x solves (H + lambda I) x = b
//   update(x, X, Xt)    Xt = X moved by the step x
// Lane 0 writes one IterStat per iteration to stats[0 ..] unless stats is null; returns the number written.  With no item included:
// no iteration, X untouched.
template <class Problem>
__device__ __forceinline__ int optimize_warp(const Problem& P, double X[Problem::N], int included, int iterations, IterStat* stats)
{
	constexpr int N = Problem::N, NSYS = N * (N + 1) / 2 + N + 1;
	if (included == 0) return 0;
	double nu = 2, lambda = 0, F = 0;
	for (int it = 0; it < iterations; it++) {
		double sys[NSYS];
#pragma unroll
		for (int i = 0; i < NSYS; i++) sys[i] = 0;
		P.linearize(sys, X);
#pragma unroll
		for (int i = 0; i < NSYS; i++) sys[i] = warp_sum(sys[i]);
		F = sys[NSYS - 1];
		if (it == 0) lambda = initial_lambda(max_diagonal<N>(sys));
		int q = 0, trials = 0;
		double rho = -1;
		for (; q < MAX_TRIALS && rho < 0; q++) {
			trials++;
			double x[N], Xt[N];
			P.solve(sys, lambda, x);
			P.update(x, X, Xt);
			const double predicted = predicted_decrease<N>(sys, lambda, x);
			const double Fhat = warp_sum(P.chi2(Xt));
			rho = gain_ratio(F, Fhat, predicted);
			if (update_damping(rho, lambda, nu)) {
				F = Fhat;
#pragma unroll
				for (int i = 0; i < N; i++) X[i] = Xt[i];
				break;
			}
		}
		if ((threadIdx.x & 31) == 0 && stats) {
			IterStat& st = stats[it];
			st.iteration = it; st.trials = trials; st.chi2 = F; st.lambda = lambda; st.pcg_iters = 0; st.pcg_failed = 0;
		}
		if (stop(q, rho, lambda)) return it + 1;
	}
	return iterations;
}

}  // namespace lm
}  // namespace cuba_b200
