// cuba_coarse.cuh -- the coarse level of both two-level PCGs (k_pcg4 in cuba_pcg4.cuh, k_pcg5 / k_pcg5t in cuba_pcg5.cuh /
// cuba_pcg5t.cuh): the basis Z_i = Ad(T_i) of every free pose, the coarse matrix Ac = Z^T S Z as a packed lower block triangle,
// and its explicit fp32 inverse.  A rebuild is k_coarse_project + k_coarse_assemble, then one of two inverses, chosen by A alone:
//   * A <= PCG4_MAXAGG1 (37): k_coarse_invert, block Cholesky + triangular inverse + W^T W in the shared memory of ONE CTA;
//   * any larger A: k_coarse_dense, a blocked symmetric sweep (block Gauss-Jordan on an SPD matrix, with every pivot applied
//     through its Cholesky factor) on the whole chip.
//
// k_coarse_dense.  A block Cholesky walks the packed 6x6-block triangle one block column at a time: A dependent diagonal
// factorisations, then the triangular inverse.  The matrix is tiny (at most 6A x 6A fp64, L2 resident) and the arithmetic is under
// a GFLOP: the time is all dependent steps.  A sweep does the work of the Cholesky factorisation, the triangular inverse and W^T W
// in one pass of 6A/32 steps over 32 x 32 scalar tiles of the dense matrix, each step spread over all SMs (one persistent
// cooperative kernel, the grid barrier of cuba_pcg2.cuh between steps).  For the pivot tile K, with A_KK = L L^T:
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

#include "cuba_pcg2.cuh"

namespace cuba_b200 {

constexpr int PCG4_MAXAGG1 = 37;    // k_coarse_invert: the packed block triangle lives in the shared memory of one CTA

// dynamic shared memory of k_coarse_invert for A aggregates: the packed blocks, the inverses of the diagonal factors, a scratch row
__host__ __device__ constexpr size_t coarse_invert_smem(int A) { return ((size_t)A * (A + 1) / 2 + 2 * (size_t)A) * 36 * sizeof(double); }

// Z_i = Ad(T_i) for every free pose: delta = [omega; upsilon], Ad = [[R, 0], [[t]x R, R]] (column-major 6x6)
template <typename T>
__global__ void k_coarse_basis(const T* __restrict__ pose, int numP, T* Zx)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= numP) return;
	const T* p = pose + 8 * (size_t)i;
	const T x = p[0], y = p[1], z = p[2], w = p[3], tx = p[4], ty = p[5], tz = p[6];
	T R[3][3];
	R[0][0] = 1 - 2 * (y * y + z * z); R[0][1] = 2 * (x * y - z * w); R[0][2] = 2 * (x * z + y * w);
	R[1][0] = 2 * (x * y + z * w); R[1][1] = 1 - 2 * (x * x + z * z); R[1][2] = 2 * (y * z - x * w);
	R[2][0] = 2 * (x * z - y * w); R[2][1] = 2 * (y * z + x * w); R[2][2] = 1 - 2 * (x * x + y * y);
	const T K[3][3] = { { T(0), -tz, ty }, { tz, T(0), -tx }, { -ty, tx, T(0) } };
	T* Z = Zx + 36 * (size_t)i;
	for (int c = 0; c < 3; c++)
		for (int r = 0; r < 3; r++) {
			Z[c * 6 + r] = R[r][c];                              // top-left R
			Z[(c + 3) * 6 + r] = T(0);                           // top-right 0
			Z[(c + 3) * 6 + r + 3] = R[r][c];                    // bottom-right R
			Z[c * 6 + r + 3] = K[r][0] * R[0][c] + K[r][1] * R[1][c] + K[r][2] * R[2][c];   // bottom-left [t]x R
		}
}

// U_n = Z_i^T S_n Z_j for every block n = (i,j) of the symmetric-full BSR: one thread per (block, entry)
template <typename T>
__global__ void k_coarse_project(const T* __restrict__ fVal, const int* __restrict__ fRowOf, const int* __restrict__ fColInd, int nfull,
	const T* __restrict__ Zx, double* U)
{
	const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= 36LL * nfull) return;
	const int n = (int)(e / 36), rc = (int)(e - 36LL * n), c = rc / 6, r = rc - 6 * c;
	const T* Sb = fVal + 36 * (size_t)n;
	const T* Zi = Zx + 36 * (size_t)fRowOf[n] + r * 6;        // column r of Z_i
	const T* Zj = Zx + 36 * (size_t)fColInd[n] + c * 6;       // column c of Z_j
	double zj[6];
#pragma unroll
	for (int m = 0; m < 6; m++) zj[m] = (double)Zj[m];
	double s = 0;
#pragma unroll
	for (int k = 0; k < 6; k++) {
		double t = 0;
#pragma unroll
		for (int m = 0; m < 6; m++) t += (double)Sb[m * 6 + k] * zj[m];      // (S Z_j)(k,c)
		s += (double)Zi[k] * t;
	}
	U[e] = s;
}

// Ac = Z^T S Z, lower block triangle, packed: block (ib >= jb) at (ib (ib+1)/2 + jb) * 36, column-major 6x6.
// cbPtr/cbList: the fine blocks of every coarse block in ascending order (built on the host) -> fixed-order sums.
__global__ void k_coarse_assemble(const int* __restrict__ cbPtr, const int* __restrict__ cbList, const double* __restrict__ U, int nblkP, double* AcP)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= nblkP * 36) return;
	const int bp = e / 36, rc = e - 36 * bp;
	double s0 = 0, s1 = 0;
	int k = cbPtr[bp];
	const int k1 = cbPtr[bp + 1];
	for (; k + 1 < k1; k += 2) { s0 += U[36 * (size_t)cbList[k] + rc]; s1 += U[36 * (size_t)cbList[k + 1] + rc]; }
	if (k < k1) s0 += U[36 * (size_t)cbList[k] + rc];
	AcP[e] = s0 + s1;
}

// AcInv = Ac^-1 by block Cholesky (6x6 blocks) of the packed lower triangle in shared memory: ONE CTA, A <= PCG4_MAXAGG1,
// coarse_invert_smem(A) bytes of dynamic shared memory.
// On a non-positive pivot the inverse is zeroed (the preconditioner degrades to block-Jacobi, still valid).
template <typename T>
__global__ void __launch_bounds__(1024, 1) k_coarse_invert(const double* __restrict__ AcP, int A, float* AcInv, int* info)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	double* B = reinterpret_cast<double*>(smem_raw);             // [nblkP][36] packed blocks
	const int nblkP = A * (A + 1) / 2, nc = 6 * A;
	double* sLi = B + (size_t)nblkP * 36;                        // [A][36] inverses of the diagonal factors
	double* sRow = sLi + (size_t)A * 36;                         // [A][36] scratch row
	__shared__ int s_fail;
	__shared__ unsigned char s_ib[PCG4_MAXAGG1 * (PCG4_MAXAGG1 + 1) / 2], s_jb[PCG4_MAXAGG1 * (PCG4_MAXAGG1 + 1) / 2];   // packed index -> (ib, jb)
	__shared__ double s_L[36], s_id[6];
	const int tid = threadIdx.x, NT = blockDim.x;
	auto idx = [](int ib, int jb) { return (size_t)(ib * (ib + 1) / 2 + jb) * 36; };
	for (int e = tid; e < nblkP * 36; e += NT) B[e] = AcP[e];
	for (int ib = tid; ib < A; ib += NT) for (int jb = 0; jb <= ib; jb++) { s_ib[ib * (ib + 1) / 2 + jb] = (unsigned char)ib; s_jb[ib * (ib + 1) / 2 + jb] = (unsigned char)jb; }
	if (tid == 0) s_fail = 0;
	__syncthreads();
	// ---- phase 1: block Cholesky, L overwrites the triangle ----
	for (int kb = 0; kb < A; kb++) {
		if (tid < 32) {
			// 6x6 Cholesky of the diagonal block in place (lane r owns row r), then L^-1 column by column (lane q owns column q)
			double* D = B + idx(kb, kb);
			const int r = tid;
			for (int j = 0; j < 6; j++) {
				const double d = D[j * 6 + j];
				if (!(d > 0)) { if (r == 0) s_fail = 1; break; }
				const double sq = sqrt(d);
				__syncwarp();
				if (r == j) D[j * 6 + j] = sq;
				else if (r > j && r < 6) D[j * 6 + r] = D[j * 6 + r] / sq;
				__syncwarp();
				if (r > j && r < 6)
					for (int c = j + 1; c <= r; c++) D[c * 6 + r] -= D[j * 6 + r] * D[j * 6 + c];
				__syncwarp();
			}
			__syncwarp();
			if (r < 6) {
				for (int c = r + 1; c < 6; c++) D[c * 6 + r] = 0.0;       // the strict upper part is not part of L
				s_id[r] = 1.0 / D[r * 6 + r];
			}
			__syncwarp();
			if (r < 6) {
				const int q = r;                                           // column q of Li = L^-1
				double col[6];
				for (int i = 0; i < 6; i++) col[i] = 0.0;
				col[q] = s_id[q];
				for (int i = q + 1; i < 6; i++) {
					double sum = 0;
					for (int k = q; k < i; k++) sum += D[k * 6 + i] * col[k];
					col[i] = -sum * s_id[i];
				}
				for (int i = 0; i < 6; i++) sLi[(size_t)kb * 36 + q * 6 + i] = col[i];
			}
		}
		__syncthreads();
		if (s_fail) break;
		// panel: B(ib,kb) <- B(ib,kb) L_kk^-T, one thread per (block, row)
		const double* Li = sLi + (size_t)kb * 36;
		for (int w = tid; w < (A - kb - 1) * 6; w += NT) {
			const int ib = kb + 1 + w / 6, r = w % 6;
			double* X = B + idx(ib, kb);
			double x[6], y[6];
			for (int k = 0; k < 6; k++) x[k] = X[k * 6 + r];
			for (int c = 0; c < 6; c++) { double s = 0; for (int k = 0; k <= c; k++) s += x[k] * Li[k * 6 + c]; y[c] = s; }   // (X Li^T)(r,c) = sum_k X(r,k) Li(c,k)
			for (int c = 0; c < 6; c++) X[c * 6 + r] = y[c];
		}
		__syncthreads();
		// trailing update: B(ib,jb) -= B(ib,kb) B(jb,kb)^T for kb < jb <= ib
		const int m = A - kb - 1;
		const int nent = m * (m + 1) / 2 * 36;
		for (int w = tid; w < nent; w += NT) {
			const int bq = w / 36, rc = w - 36 * bq, c = rc / 6, r = rc - 6 * c;
			const int ib = kb + 1 + s_ib[bq], jb = kb + 1 + s_jb[bq];
			const double* P = B + idx(ib, kb);
			const double* Q = B + idx(jb, kb);
			double s = 0;
			for (int k = 0; k < 6; k++) s += P[k * 6 + r] * Q[k * 6 + c];
			B[idx(ib, jb) + c * 6 + r] -= s;
		}
		__syncthreads();
	}
	if (s_fail) {
		for (int e = tid; e < nc * nc; e += NT) AcInv[e] = 0.f;
		if (tid == 0 && info) *info = 1;
		return;
	}
	// ---- phase 2: W = L^-1 (block lower triangular), row by row: W(ib,jb) = -L_ii^-1 sum_{k=jb}^{ib-1} L(ib,k) W(k,jb) ----
	for (int ib = 0; ib < A; ib++) {
		for (int w = tid; w < ib * 36; w += NT) {
			const int jb = w / 36, rc = w - 36 * jb, c = rc / 6, r = rc - 6 * c;
			double s = 0;
			for (int k = jb; k < ib; k++) {
				const double* Lb = B + idx(ib, k);
				const double* Wb = B + idx(k, jb);               // rows < ib already hold W (diagonal blocks: W(k,k) = L_kk^-1)
				for (int mm = 0; mm < 6; mm++) s += Lb[mm * 6 + r] * Wb[c * 6 + mm];
			}
			sRow[(size_t)jb * 36 + c * 6 + r] = s;
		}
		__syncthreads();
		const double* Li = sLi + (size_t)ib * 36;
		for (int w = tid; w < (ib + 1) * 36; w += NT) {
			const int jb = w / 36, rc = w - 36 * jb, c = rc / 6, r = rc - 6 * c;
			double v;
			if (jb == ib) v = Li[c * 6 + r];
			else {
				double s = 0;
				for (int k = 0; k <= r; k++) s += Li[k * 6 + r] * sRow[(size_t)jb * 36 + c * 6 + k];   // Li lower: Li(r,k), k <= r
				v = -s;
			}
			B[idx(ib, jb) + c * 6 + r] = v;
		}
		__syncthreads();
	}
	// ---- phase 3: Ac^-1 = W^T W; block (ib,jb), ib >= jb: sum_{k >= ib} W(k,ib)^T W(k,jb) ----
	for (int w = tid; w < nblkP * 36; w += NT) {
		const int bq = w / 36, rc = w - 36 * bq, c = rc / 6, r = rc - 6 * c;
		const int ib = s_ib[bq], jb = s_jb[bq];
		double s = 0;
		for (int k = ib; k < A; k++) {
			const double* Wa = B + idx(k, ib);
			const double* Wb = B + idx(k, jb);
			for (int mm = 0; mm < 6; mm++) s += Wa[r * 6 + mm] * Wb[c * 6 + mm];
		}
		AcInv[(size_t)(ib * 6 + r) * nc + jb * 6 + c] = (float)s;
		AcInv[(size_t)(jb * 6 + c) * nc + ib * 6 + r] = (float)s;
	}
	if (tid == 0 && info) *info = 0;
}

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
// doubles of Args::T for A aggregates
inline size_t scratch_doubles(int A) { return 2 * tiles((6 * A + NB - 1) / NB) * TT; }
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
