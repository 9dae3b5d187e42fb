// cuba_coarse_dense.cuh -- explicit inverse of the coarse matrix Ac = Z^T S Z of the two-level PCG (cuba_pcg5.cuh) by a blocked
// symmetric sweep (block Gauss-Jordan on an SPD matrix, with every pivot applied through its Cholesky factor) on the whole chip.
//
// The cluster kernels of cuba_pcg4.cuh keep the packed 6x6-block triangle in the shared memory of 8 / 16 CTAs and walk it one
// block column at a time: A aggregates = A x (diagonal factorisation by one warp + two cluster barriers), plus the triangular
// inverse.  The matrix is tiny (at most 6A x 6A fp64, L2 resident) and the arithmetic is under a GFLOP: the time is all dependent
// steps.  A sweep does the work of the Cholesky factorisation, the triangular inverse and W^T W in one pass of 6A/32 steps over
// 32 x 32 scalar tiles of the dense matrix, each step spread over all SMs (one persistent cooperative kernel, the grid barrier of
// cuba_pcg2.cuh between steps).  For the pivot tile K, with A_KK = L L^T:
//     Q_I   = A_IK L^-T                      every I != K
//     A_IJ -= Q_I Q_J^T                      every lower tile I >= J, I, J != K
//     A_IK  = Q_I L^-1,  A_KK = -L^-T L^-1
// and after the last step A = -Ac^-1.  The update is applied as Q_I Q_J^T, never through the explicit P = A_KK^-1: on the
// coarse matrix of rows_11k at lambda 0.1 (condition ~1e15, most of it scaling) A_IK P A_KJ loses the inverse to 4e-5 of its
// largest entry, the factored form keeps it at 2e-8, as a Cholesky inverse does.  Only the lower tiles are kept (A_KJ = A_JK^T), so
// the result is symmetric by construction; diagonal tiles are mirrored from their lower triangle whenever they are stored.
//   phase 0  packed blocks -> lower tiles of copy 0 (padded to a multiple of 32 with a unit diagonal);
//   step K   reads copy K & 1 and writes copy (K + 1) & 1, every lower tile, so that nothing is read after it is rewritten;
//            every CTA factors the pivot tile itself in registers (warp 0: 32 scalar Cholesky steps, then L^-1 by forward
//            substitution, no hop) while its warps stage their tiles; one WARP per trailing tile forms Q_I and Q_J on the fp64
//            tensor pipe (redundant across the tiles of a row, but it removes the panel barrier) and updates its tile, and the warp
//            of tile (I, I) also stores Q_I L^-1 as the new panel tile;  ONE grid barrier per step;  the last step writes -A in
//            fp32 to both triangles of Ac^-1 (the PCG applies it in fp32, see cuba_pcg4.cuh) instead of a copy.
// Fixed summation order everywhere, no atomics: bit-reproducible.  On a non-positive pivot the inverse is zeroed (block-Jacobi
// alone).
#pragma once

#include "cuba_pcg4.cuh"

namespace cuba_b200 {
namespace cdense {

constexpr int NB = 32;                 // tile edge
constexpr int TT = NB * NB;            // doubles per stored tile (row-major)
constexpr int WARPS = 8;
constexpr int TS = NB + 4;             // row stride of a staged tile: the fragment loads of both orientations hit 16 distinct banks
constexpr size_t SMEM = ((size_t)(2 * WARPS + 2) * NB * TS + NB) * sizeof(double);

struct Args {
	const double* AcP;                 // packed lower block triangle, block (ib >= jb) at (ib (ib+1)/2 + jb) * 36, column-major 6x6
	int A;                             // aggregates: n = 6 A
	double* T;                         // [2][nt (nt+1) / 2][NB * NB] two copies of the lower tiles, tile (I >= J) at I (I+1)/2 + J
	float* AcInv;                      // [n][n] out
	int* info;                         // 0 ok, 1 not positive definite
	GridBar* bar;
};

__host__ __device__ constexpr size_t tiles(int nt) { return (size_t)nt * (nt + 1) / 2; }
__device__ __forceinline__ const double* tile(const double* C, int I, int J) { return C + ((size_t)I * (I + 1) / 2 + J) * TT; }
__device__ __forceinline__ double* tile(double* C, int I, int J) { return C + ((size_t)I * (I + 1) / 2 + J) * TT; }

// t -> (i, j), i >= j, of the lower triangle enumerated row by row
__device__ __forceinline__ void tri_decode(int t, int& i, int& j)
{
	i = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
	while ((i + 1) * (i + 2) / 2 <= t) i++;
	while (i * (i + 1) / 2 > t) i--;
	j = t - i * (i + 1) / 2;
}

// one warp copies a stored tile into shared memory (row stride TS) with 16-byte cp.async through L2
__device__ __forceinline__ void stage(double* s, const double* g, int lane)
{
#pragma unroll
	for (int e = lane; e < TT / 2; e += 32) {
		const int r = e >> 4, c = (e & 15) * 2;
		cp_async16(s + r * TS + c, g + r * NB + c);
	}
	asm volatile("cp.async.commit_group;" ::: "memory");
}

// 32 x 32 x 32 product on the fp64 tensor pipe: D(8 bi + l/4, 8 bj + 2 (l%4) + h) += sum_m X(row, m) Y(m, col), with
// X(r, m) = sX[r * xr + m * xc] and Y(m, c) = sY[m * yr + c * yc]; the k-steps in order
__device__ __forceinline__ void mma32(double (&D)[4][4][2], const double* sX, int xr, int xc, const double* sY, int yr, int yc, int lane)
{
	const int r = lane >> 2, q = lane & 3;
	const double* xb = sX + r * xr + q * xc;
	const double* yb = sY + q * yr + r * yc;
#pragma unroll
	for (int s = 0; s < NB / 4; s++) {
		double a[4], b[4];
#pragma unroll
		for (int u = 0; u < 4; u++) { a[u] = xb[8 * u * xr + 4 * s * xc]; b[u] = yb[4 * s * yr + 8 * u * yc]; }
#pragma unroll
		for (int bi = 0; bi < 4; bi++)
#pragma unroll
			for (int bj = 0; bj < 4; bj++) dmma884(D[bi][bj][0], D[bi][bj][1], a[bi], b[bj]);
	}
}

// sgn x accumulator fragments -> shared memory (row-major, stride TS)
__device__ __forceinline__ void frag_store(double* s, const double (&D)[4][4][2], double sgn, int lane)
{
	const int r = lane >> 2, c = 2 * (lane & 3);
#pragma unroll
	for (int bi = 0; bi < 4; bi++)
#pragma unroll
		for (int bj = 0; bj < 4; bj++) *reinterpret_cast<double2*>(s + (8 * bi + r) * TS + 8 * bj + c) = make_double2(sgn * D[bi][bj][0], sgn * D[bi][bj][1]);
}

// a finished tile in shared memory (element (r, c) = sgn s[r * sr + c * sc]; a diagonal tile mirrored from its lower triangle)
// -> tile (I, J) of the next copy, or, at the last step, -value in fp32 to both triangles of Ac^-1
__device__ __forceinline__ void tile_out(const double* s, int sr, int sc, double sgn, bool diag, int I, int J, double* dst, bool last,
                                         float* AcInv, int n, int lane)
{
	auto at = [&](int r, int c) { if (diag && r < c) { const int t = r; r = c; c = t; } return sgn * s[r * sr + c * sc]; };
	if (!last) {
		for (int e = lane; e < TT / 2; e += 32) {
			const int r = e >> 4, c = (e & 15) * 2;
			__stcg(reinterpret_cast<double2*>(dst + r * NB + c), make_double2(at(r, c), at(r, c + 1)));
		}
		return;
	}
	for (int e = lane; e < TT; e += 32) {
		const int r = e >> 5, c = e & 31;
		const int row = NB * I + r, col = NB * J + c;
		if (row < n && col < n) AcInv[(size_t)row * n + col] = (float)-at(r, c);
		const int row2 = NB * J + r, col2 = NB * I + c;                  // mirror: element (c, r) of the tile
		if (I != J && row2 < n && col2 < n) AcInv[(size_t)row2 * n + col2] = (float)-at(c, r);
	}
}

__global__ void __launch_bounds__(WARPS * 32, 1) k_coarse_dense(const Args a)
{
	extern __shared__ __align__(16) double smem[];
	double* sN = smem;                                 // L^-1 of this step's pivot (lower), row-major, stride TS
	double* sPv = sN + NB * TS;                        // warp 0: L, then -P of CTA 0
	double* sRow = sPv + NB * TS;                      // warp 0: a column of L / the reciprocals of its diagonal
	double* sW = sRow + NB;                            // [WARPS][2][NB * TS] per warp: two staged tiles
	__shared__ int s_fail;
	__shared__ unsigned int s_gen;
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	const int G = gridDim.x, cta = blockIdx.x;
	const int n = 6 * a.A, nt = (n + NB - 1) / NB;
	if (tid == 0) { s_gen = ld_acquire_u32(&a.bar->gen); s_fail = 0; }
	__syncthreads();
	unsigned int gen = s_gen;

	// ---- phase 0: packed 6x6 blocks -> lower tiles of copy 0 (lower triangle of the diagonal blocks); unit diagonal in the padding ----
	{
		const long long tot = (long long)tiles(nt) * TT;
		for (long long e = (long long)cta * blockDim.x + tid; e < tot; e += (long long)G * blockDim.x) {
			const int t = (int)(e / TT), rc = (int)(e - (long long)t * TT);
			int I, J;
			tri_decode(t, I, J);
			int row = NB * I + (rc >> 5), col = NB * J + (rc & 31);
			if (row < col) { const int x = row; row = col; col = x; }
			double v = row == col ? 1.0 : 0.0;
			if (row < n) {
				const int ib = row / 6, jb = col / 6;
				v = a.AcP[((size_t)ib * (ib + 1) / 2 + jb) * 36 + (col - 6 * jb) * 6 + (row - 6 * ib)];
			}
			__stcg(a.T + e, v);
		}
	}
	grid_barrier(a.bar, G, gen);

	double* sA = sW + (size_t)wid * 2 * NB * TS;
	double* sB = sA + NB * TS;
	const int slot = (wid + WARPS - 1) % WARPS;         // warp 0 factors the pivot: it takes a tile last
	const int m = nt - 1, ntl = m * (m + 1) / 2;         // trailing tiles per step
	for (int K = 0; K < nt; K++) {
		const double* src = a.T + (size_t)(K & 1) * tiles(nt) * TT;
		double* dst = a.T + (size_t)((K + 1) & 1) * tiles(nt) * TT;
		const bool last = K == nt - 1;
		int t = slot * G + cta;
		int I = 0, J = 0;
		auto locate = [&](int tt) {
			int li, lj;
			tri_decode(tt, li, lj);
			I = li + (li >= K); J = lj + (lj >= K);
		};
		// A_XK of the step: tile (X, K) below the pivot, the transpose of tile (K, X) above it
		auto issue = [&]() {
			stage(sA, I > K ? tile(src, I, K) : tile(src, K, I), lane);
			stage(sB, J > K ? tile(src, J, K) : tile(src, K, J), lane);
		};
		if (t < ntl) { locate(t); issue(); }
		if (wid == 0) {
			// ---- the pivot: every CTA factors A_KK = L L^T in registers (lane i holds row i) and forms L^-1 (lane q: column q) ----
			double row[NB];
			const double* g = tile(src, K, K) + lane * NB;
#pragma unroll
			for (int i = 0; i < NB; i += 2) { const double2 v = __ldcg(reinterpret_cast<const double2*>(g + i)); row[i] = v.x; row[i + 1] = v.y; }
			bool ok = true;
			double rdiag = 0.0;                          // lane i: 1 / L(i, i)
#pragma unroll
			for (int k = 0; k < NB; k++) {
				sRow[lane] = row[k];
				__syncwarp();
				const double d = sRow[k];
				if (!(d > 0)) { ok = false; break; }
				const double lkk = sqrt(d), rk = 1.0 / lkk;
				const double lik = lane > k ? row[k] * rk : lane == k ? lkk : 0.0;      // column k of L
				if (lane == k) rdiag = rk;
				__syncwarp();
				sRow[lane] = lik;
				__syncwarp();
#pragma unroll
				for (int j = k + 1; j < NB; j++) row[j] = fma(-lik, sRow[j], row[j]);
				row[k] = lik;
				__syncwarp();
			}
			if (!ok) { if (lane == 0) s_fail = 1; }
			else {
				// row = row `lane` of L (lower); column q of L^-1 by forward substitution, x_i = (delta_iq - sum_{k<i} L_ik x_k) / L_ii
#pragma unroll
				for (int i = 0; i < NB; i += 2) *reinterpret_cast<double2*>(sPv + lane * TS + i) = make_double2(row[i], row[i + 1]);
				sRow[lane] = rdiag;
				__syncwarp();
				double x[NB];
#pragma unroll
				for (int i = 0; i < NB; i++) {
					double sum = i == lane ? 1.0 : 0.0;
#pragma unroll
					for (int k = 0; k < i; k++) sum = fma(-sPv[i * TS + k], x[k], sum);
					x[i] = sum * sRow[i];
				}
#pragma unroll
				for (int i = 0; i < NB; i++) sN[i * TS + lane] = x[i];
				__syncwarp();
				if (cta == 0) {
					// the new pivot tile -P = -L^-T L^-1
					double pp[4][4][2];
#pragma unroll
					for (int bi = 0; bi < 4; bi++)
#pragma unroll
						for (int bj = 0; bj < 4; bj++) pp[bi][bj][0] = pp[bi][bj][1] = 0.0;
					mma32(pp, sN, 1, TS, sN, TS, 1, lane);
					frag_store(sPv, pp, 1.0, lane);
					__syncwarp();
					tile_out(sPv, TS, 1, -1.0, true, K, K, tile(dst, K, K), last, a.AcInv, n, lane);
				}
			}
		}
		__syncthreads();
		if (s_fail) { asm volatile("cp.async.wait_group 0;" ::: "memory"); break; }   // every CTA sees the same pivots

		for (bool first = true; t < ntl; t += G * WARPS, first = false) {
			if (!first) { locate(t); issue(); }
			const bool trI = I < K, trJ = J < K;
			// acc = A_IJ (fragment layout), from the copy of this step
			double acc[4][4][2];
			{
				const double* g = tile(src, I, J) + (lane >> 2) * NB + 2 * (lane & 3);
#pragma unroll
				for (int bi = 0; bi < 4; bi++)
#pragma unroll
					for (int bj = 0; bj < 4; bj++) {
						const double2 v = __ldcg(reinterpret_cast<const double2*>(g + 8 * bi * NB + 8 * bj));
						acc[bi][bj][0] = v.x; acc[bi][bj][1] = v.y;
					}
			}
			asm volatile("cp.async.wait_group 0;" ::: "memory");
			__syncwarp();
			// Q_I = A_IK L^-T into sA over A_IK; -Q_J = -A_JK L^-T into sB over A_JK (tile (I, I): -Q_I)
			double q[4][4][2];
#pragma unroll
			for (int bi = 0; bi < 4; bi++)
#pragma unroll
				for (int bj = 0; bj < 4; bj++) q[bi][bj][0] = q[bi][bj][1] = 0.0;
			mma32(q, sA, trI ? 1 : TS, trI ? TS : 1, sN, 1, TS, lane);
			__syncwarp();
			frag_store(sA, q, 1.0, lane);
			if (I == J) frag_store(sB, q, -1.0, lane);
			else {
#pragma unroll
				for (int bi = 0; bi < 4; bi++)
#pragma unroll
					for (int bj = 0; bj < 4; bj++) q[bi][bj][0] = q[bi][bj][1] = 0.0;
				mma32(q, sB, trJ ? 1 : TS, trJ ? TS : 1, sN, 1, TS, lane);
				__syncwarp();
				frag_store(sB, q, -1.0, lane);
			}
			__syncwarp();
			// A_IJ - A_IK P A_KJ = A_IJ - Q_I Q_J^T
			mma32(acc, sA, TS, 1, sB, 1, TS, lane);
			if (I == J) {
				// the warp of tile (I, I) also forms the new panel tile A_IK P = Q_I L^-1
#pragma unroll
				for (int bi = 0; bi < 4; bi++)
#pragma unroll
					for (int bj = 0; bj < 4; bj++) q[bi][bj][0] = q[bi][bj][1] = 0.0;
				mma32(q, sA, TS, 1, sN, TS, 1, lane);
			}
			__syncwarp();
			frag_store(sB, acc, 1.0, lane);
			__syncwarp();
			tile_out(sB, TS, 1, 1.0, I == J, I, J, tile(dst, I, J), last, a.AcInv, n, lane);
			__syncwarp();
			if (I == J) {
				// tile (I, K) below the pivot, or its transpose, tile (K, I), above it
				frag_store(sB, q, 1.0, lane);
				__syncwarp();
				if (I > K) tile_out(sB, TS, 1, 1.0, false, I, K, tile(dst, I, K), last, a.AcInv, n, lane);
				else tile_out(sB, 1, TS, 1.0, false, K, I, tile(dst, K, I), last, a.AcInv, n, lane);
				__syncwarp();
			}
		}
		if (!last) grid_barrier(a.bar, G, gen);
	}
	if (s_fail) {
		for (long long e = (long long)cta * blockDim.x + tid; e < (long long)n * n; e += (long long)G * blockDim.x) a.AcInv[e] = 0.f;
		if (cta == 0 && tid == 0) *a.info = 1;
		return;
	}
	if (cta == 0 && tid == 0) *a.info = 0;
}

}  // namespace cdense
}  // namespace cuba_b200
