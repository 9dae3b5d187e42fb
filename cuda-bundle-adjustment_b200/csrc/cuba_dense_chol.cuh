// cuba_dense_chol.cuh -- the direct solver of the reduced camera system (cuba_engine_set_linear_solver(CUBA_SOLVER_DENSE_CHOLESKY)):
// S xp = bsc by a dense Cholesky factorisation S = L L^T on the fp64 tensor pipe, in ONE persistent cooperative kernel.
//
// S (symmetric-full BSR of the Schur stage, lambda already on the diagonal) is scattered into the lower 32 x 32 tiles of the padded
// n x n matrix (n = 6 numP, padded to a multiple of 32 with a unit diagonal), always in fp64: the fp32 engine's blocks are widened.
// The tile layout and helpers are those of k_coarse_dense (cuba_coarse.cuh, namespace cdense).  Right-looking blocked Cholesky, per
// pivot tile K, with two grid barriers:
//   panel   every CTA factors A_KK = L_KK L_KK^T in registers (warp 0, cdense::pivot_factor); one warp per tile I > K solves
//           L_IK L_KK^T = A_IK by substitution, in place; one more warp forms y_K = L_KK^-1 y_K (forward substitution, y = bsc)
//   update  one warp per trailing tile K < J <= I:  A_IJ -= L_IK L_JK^T  (DMMA m8n8k4, cdense::mma32); the warp of tile (I, I) also
//           applies y_I -= L_IK y_K; CTA 0 stores L_KK into tile (K, K)
// Within a phase every tile is read and written by one warp only, and nothing a phase reads is rewritten in it.  Then the backward
// substitution L^T x = y, one grid barrier per tile row K (descending): every warp with an item forms x_K = L_KK^-T y_K itself, the
// item J < K applies y_J -= L_KJ^T x_K, the item J = K writes x_K (in T).
// Triangular solves are substitutions (no explicit inverse), so Cholesky's backward-error bound holds.  Fixed summation order, no
// atomics: bit-reproducible.  A pivot that is not positive stops every CTA at the same step (all factor the same tile): x = 0,
// status 2 (info 1).
#pragma once

#include "cuba_coarse.cuh"

namespace cuba_b200 {
namespace dchol {

using cdense::NB;
using cdense::TT;
using cdense::TS;
using cdense::WARPS;

constexpr int MAX_POSES = 2730;        // n <= 16380: 512 tile rows, 1.08 GB of lower tiles
// L_KK (stride TS), 1 / diag(L_KK), and two staged tiles per warp
constexpr size_t SMEM = ((size_t)(2 * WARPS + 1) * NB * TS + NB) * sizeof(double);

__host__ __device__ constexpr int tile_rows(int n) { return (n + NB - 1) / NB; }
// doubles of Args::tl and of Args::y for an n x n system
inline size_t tile_doubles(int n) { return cdense::tiles(tile_rows(n)) * TT; }
inline size_t rhs_doubles(int n) { return (size_t)tile_rows(n) * NB; }

template <typename T>
struct Args {
	const T* fVal;            // symmetric-full BSR blocks (column-major 6x6) ...
	const int* blkMap;        // ... reached through the packed lower block triangle: block (i >= j) at i (i+1)/2 + j, -1 = none
	const double* dense;      // or, when not null, a row-major n x n matrix (cuba_debug_dense_solve)
	const T* b;               // [n]
	int n;
	double* tl;               // [tiles(nt)][NB * NB] lower tiles, tile (I >= J) at I (I+1)/2 + J, row-major
	double* y;                // [nt NB] right-hand side, then L^-1 b
	T* x;                     // [n] out
	PcgStatus* status;        // the engine's solver slot (iters 0; status 0, or 2 when S is not positive definite), or null
	int* info;                // 0, or 1 when S is not positive definite; or null
	GridBar* bar;
};

template <typename T>
__global__ void __launch_bounds__(WARPS * 32, 1) k_dense_chol(const Args<T> a)
{
	extern __shared__ __align__(16) double smem[];
	double* sL = smem;                                 // L_KK of this step, row-major, stride TS
	double* sD = sL + NB * TS;                         // its reciprocal diagonal (warp 0's scratch while it factors)
	double* sW = sD + NB;                              // [WARPS][2][NB * TS] per warp: two staged tiles
	__shared__ int s_fail;
	__shared__ unsigned int s_gen;
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	const int G = gridDim.x, cta = blockIdx.x;
	const int gw = wid * G + cta, NW = G * WARPS;      // this warp among all warps (consecutive items go to different CTAs)
	const int n = a.n, nt = tile_rows(n);
	constexpr unsigned FULL = 0xffffffffu;
	if (tid == 0) { s_gen = ld_acquire_u32(&a.bar->gen); s_fail = 0; }
	__syncthreads();
	unsigned int gen = s_gen;

	// ---- scatter: S -> lower tiles (the lower triangle of the diagonal tiles mirrored), unit diagonal in the padding; b -> y ----
	{
		const long long tot = (long long)cdense::tiles(nt) * TT;
		for (long long e = (long long)cta * blockDim.x + tid; e < tot; e += (long long)G * blockDim.x) {
			const int t = (int)(e / TT), rc = (int)(e - (long long)t * TT);
			int I, J;
			cdense::tri_decode(t, I, J);
			int row = NB * I + (rc >> 5), col = NB * J + (rc & 31);
			if (row < col) { const int s = row; row = col; col = s; }
			double v = row == col ? 1.0 : 0.0;
			if (row < n) {
				if (a.dense) v = a.dense[(size_t)row * n + col];
				else {
					const int ib = row / 6, jb = col / 6;
					const int m = a.blkMap[(size_t)ib * (ib + 1) / 2 + jb];
					v = m < 0 ? 0.0 : (double)a.fVal[36 * (size_t)m + (col - 6 * jb) * 6 + (row - 6 * ib)];
				}
			}
			__stcg(a.tl + e, v);
		}
		for (int i = cta * blockDim.x + tid; i < nt * NB; i += G * blockDim.x) __stcg(a.y + i, i < n ? (double)a.b[i] : 0.0);
	}
	grid_barrier(a.bar, G, gen);

	double* sA = sW + (size_t)wid * 2 * NB * TS;
	double* sB = sA + NB * TS;
	for (int K = 0; K < nt; K++) {
		// ---- panel: the pivot in every CTA, then L_IK = A_IK L_KK^-T per tile and y_K = L_KK^-1 y_K ----
		if (wid == 0) {
			double row[NB];
			double rdiag;
			if (!cdense::pivot_factor(cdense::tile(a.tl, K, K), row, rdiag, sD, lane)) { if (lane == 0) s_fail = 1; }
			else {
#pragma unroll
				for (int i = 0; i < NB; i += 2) *reinterpret_cast<double2*>(sL + lane * TS + i) = make_double2(row[i], row[i + 1]);
				__syncwarp();
				sD[lane] = rdiag;
			}
		}
		__syncthreads();
		if (s_fail) break;                             // every CTA sees the same pivot
		const int np = nt - 1 - K;
		for (int p = gw; p <= np; p += NW) {
			if (p < np) {
				// lane r: row r of A_IK; x_j = (a_j - sum_{k<j} x_k L(j, k)) / L(j, j)
				double* g = cdense::tile(a.tl, K + 1 + p, K) + lane * NB;
				double r[NB];
#pragma unroll
				for (int i = 0; i < NB; i += 2) { const double2 v = __ldcg(reinterpret_cast<const double2*>(g + i)); r[i] = v.x; r[i + 1] = v.y; }
#pragma unroll
				for (int j = 0; j < NB; j++) {
					double s = r[j];
#pragma unroll
					for (int k = 0; k < j; k++) s = fma(-r[k], sL[j * TS + k], s);
					r[j] = s * sD[j];
				}
#pragma unroll
				for (int i = 0; i < NB; i += 2) __stcg(reinterpret_cast<double2*>(g + i), make_double2(r[i], r[i + 1]));
			} else {
				// forward substitution L_KK y_K = b_K: lane i holds entry i
				double v = __ldcg(a.y + (size_t)K * NB + lane);
#pragma unroll
				for (int k = 0; k < NB; k++) {
					const double yk = __shfl_sync(FULL, v, k) * sD[k];
					if (lane > k) v = fma(-sL[lane * TS + k], yk, v);
					else if (lane == k) v = yk;
				}
				__stcg(a.y + (size_t)K * NB + lane, v);
			}
		}
		grid_barrier(a.bar, G, gen);

		// ---- update: A_IJ -= L_IK L_JK^T for K < J <= I, y_I -= L_IK y_K ----
		if (cta == 0 && wid == 0) {
			double* g = cdense::tile(a.tl, K, K);
			for (int e = lane; e < TT / 2; e += 32) {
				const int r = e >> 4, c = (e & 15) * 2;
				__stcg(reinterpret_cast<double2*>(g + r * NB + c), make_double2(sL[r * TS + c], sL[r * TS + c + 1]));
			}
		}
		const int ntl = np * (np + 1) / 2;
		for (int t = gw; t < ntl; t += NW) {
			int li, lj;
			cdense::tri_decode(t, li, lj);
			const int I = K + 1 + li, J = K + 1 + lj;
			cdense::stage(sA, cdense::tile(a.tl, I, K), lane);
			if (I != J) cdense::stage(sB, cdense::tile(a.tl, J, K), lane);
			const double* sJ = I != J ? sB : sA;
			double acc[4][4][2];                       // -A_IJ in fragment layout
			{
				const double* g = cdense::tile(a.tl, I, J) + (lane >> 2) * NB + 2 * (lane & 3);
#pragma unroll
				for (int bi = 0; bi < 4; bi++)
#pragma unroll
					for (int bj = 0; bj < 4; bj++) {
						const double2 v = __ldcg(reinterpret_cast<const double2*>(g + 8 * bi * NB + 8 * bj));
						acc[bi][bj][0] = -v.x; acc[bi][bj][1] = -v.y;
					}
			}
			asm volatile("cp.async.wait_group 0;" ::: "memory");
			__syncwarp();
			cdense::mma32(acc, sA, TS, 1, sJ, 1, TS, lane);
			__syncwarp();
			cdense::frag_store(sB, acc, -1.0, lane);
			__syncwarp();
			double* g = cdense::tile(a.tl, I, J);
			for (int e = lane; e < TT / 2; e += 32) {
				const int r = e >> 4, c = (e & 15) * 2;
				__stcg(reinterpret_cast<double2*>(g + r * NB + c), make_double2(sB[r * TS + c], sB[r * TS + c + 1]));
			}
			if (I == J) {
				double s = 0.0;
#pragma unroll
				for (int k = 0; k < NB; k++) s = fma(sA[lane * TS + k], __ldcg(a.y + (size_t)K * NB + k), s);
				double* yi = a.y + (size_t)I * NB + lane;
				__stcg(yi, __ldcg(yi) - s);
			}
			__syncwarp();
		}
		grid_barrier(a.bar, G, gen);
	}

	if (s_fail) {
		for (int i = cta * blockDim.x + tid; i < n; i += G * blockDim.x) a.x[i] = T(0);
		if (cta == 0 && tid == 0) {
			if (a.status) { a.status->iters = 0; a.status->status = 2; a.status->rz0 = 0; a.status->rz = 0; }
			if (a.info) *a.info = 1;
		}
		return;
	}

	// ---- backward substitution L^T x = y, one tile row per step ----
	for (int K = nt - 1; K >= 0; K--) {
		for (int j = gw; j <= K; j += NW) {
			cdense::stage(sA, cdense::tile(a.tl, K, K), lane);
			if (j < K) cdense::stage(sB, cdense::tile(a.tl, K, j), lane);
			double v = __ldcg(a.y + (size_t)K * NB + lane);
			asm volatile("cp.async.wait_group 0;" ::: "memory");
			__syncwarp();
			const double rd = 1.0 / sA[lane * TS + lane];
#pragma unroll
			for (int k = NB - 1; k >= 0; k--) {
				const double xk = __shfl_sync(FULL, v, k) * __shfl_sync(FULL, rd, k);
				if (lane < k) v = fma(-sA[k * TS + lane], xk, v);
				else if (lane == k) v = xk;
			}
			if (j == K) {
				const int i = K * NB + lane;
				if (i < n) a.x[i] = (T)v;
			} else {
				__syncwarp();
				sA[lane] = v;                          // x_K over row 0 of L_KK (no longer needed)
				__syncwarp();
				double s = 0.0;
#pragma unroll
				for (int r = 0; r < NB; r++) s = fma(sB[r * TS + lane], sA[r], s);
				double* yj = a.y + (size_t)j * NB + lane;
				__stcg(yj, __ldcg(yj) - s);
			}
			__syncwarp();
		}
		if (K > 0) grid_barrier(a.bar, G, gen);
	}
	if (cta == 0 && tid == 0) {
		if (a.status) { a.status->iters = 0; a.status->status = 0; a.status->rz0 = 0; a.status->rz = 0; }
		if (a.info) *a.info = 0;
	}
}

}  // namespace dchol
}  // namespace cuba_b200
