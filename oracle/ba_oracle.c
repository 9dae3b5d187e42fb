/*
 * ba_oracle.c -- CPU restatement of the reference's LM bundle adjustment (fp64).
 *
 * TEST INFRASTRUCTURE ONLY (see ba_oracle.h).  Plain C99, single file, no dependencies.
 * The Schur system is solved with a direct sparse block Cholesky (minimum-degree ordered), i.e.
 * the same mathematics as the reference's cuSOLVER csrchol (src/cuda_linear_solver.cpp:301-335)
 * and g2o's LinearSolverEigen; it is NOT the product's PCG.
 *
 * Parity: pinned against README.md:141-150 (see tests/test_oracle_golden.py).
 */
#include "ba_oracle.h"

#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define PD 6
#define LD 3

struct bao {
	int Pall, numP, Lall, numL, E2, E3, E;
	int rk_type[2];
	double rk_delta[2];
	/* state (src/cuda_bundle_adjustment.cpp:322-331) + backup (push/pop :502-510) */
	double *q, *t, *cam, *Xw, *q_bak, *t_bak, *Xw_bak;
	/* edges, edge id order: mono then stereo (cpp:203-243) */
	int* ePL;          /* [2E] */
	double* meas;      /* [3E] (mono uses 2) */
	double* omega;     /* [E] */
	unsigned char* flag; /* [E] EDGE_FLAG_FIXED_L=1, EDGE_FLAG_FIXED_P=2 (src/constants.h:32-36) */
	double* err;       /* [3E] */
	double* Xc;        /* [3E] */
	/* structure */
	int nhpl, nblk, nmul;
	int *hplColPtr, *hplRowInd, *edge2Hpl, *hplEdge; /* CSC of Hpl (cu:1158-1173) */
	int *hscRowPtr, *hscColInd;                     /* upper BSR of Hsc (sparse_block_matrix.cpp:55-133) */
	/* linear system */
	double *Hpp, *bp, *Hll, *bl, *Hpl;
	double *Hsc, *bsc, *invHll, *xp, *xl;
	/* block Cholesky workspace */
	int* perm;      /* elimination order: perm[k] = original block index eliminated k-th */
	int* iperm;
	int* Lptr;      /* [numP+1] column pointers (in eliminated order) into Lrow/Lval */
	int* Lrow;      /* row (elimination positions), first entry of each column is the diagonal */
	double* Lval;   /* 36 per block */
	int* posmap;    /* scratch [numP] */
	int chol_ready;
};

/* ---------------------------------------------------------------- small dense helpers */

/* cu:245-260 rotate(): Xc = R(q) * X via two cross products */
static void rotate(const double* q, const double* X, double* Xc)
{
	double t1[3], t2[3];
	t1[0] = q[1] * X[2] - q[2] * X[1];
	t1[1] = q[2] * X[0] - q[0] * X[2];
	t1[2] = q[0] * X[1] - q[1] * X[0];
	t1[0] += t1[0]; t1[1] += t1[1]; t1[2] += t1[2];
	t2[0] = q[1] * t1[2] - q[2] * t1[1];
	t2[1] = q[2] * t1[0] - q[0] * t1[2];
	t2[2] = q[0] * t1[1] - q[1] * t1[0];
	Xc[0] = X[0] + q[3] * t1[0] + t2[0];
	Xc[1] = X[1] + q[3] * t1[1] + t2[1];
	Xc[2] = X[2] + q[3] * t1[2] + t2[2];
}

/* cu:262-268 */
static void project_w2c(const double* q, const double* t, const double* Xw, double* Xc)
{
	rotate(q, Xw, Xc);
	Xc[0] += t[0]; Xc[1] += t[1]; Xc[2] += t[2];
}

/* cu:275-290 */
static void project_c2i(const double* Xc, const double* cam, int mdim, double* p)
{
	const double invZ = 1 / Xc[2];
	p[0] = cam[0] * invZ * Xc[0] + cam[2];
	p[1] = cam[1] * invZ * Xc[1] + cam[3];
	if (mdim == 3)
		p[2] = p[0] - cam[4] * invZ;
}

/* cu:292-321, column-major 3x3 */
static void quat_to_rot(const double* q, double* R)
{
	const double x = q[0], y = q[1], z = q[2], w = q[3];
	const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
	const double twx = tx * w, twy = ty * w, twz = tz * w;
	const double txx = tx * x, txy = ty * x, txz = tz * x;
	const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
#define R_(i, j) R[(j) * 3 + (i)]
	R_(0, 0) = 1 - (tyy + tzz); R_(0, 1) = txy - twz;       R_(0, 2) = txz + twy;
	R_(1, 0) = txy + twz;       R_(1, 1) = 1 - (txx + tzz); R_(1, 2) = tyz - twx;
	R_(2, 0) = txz - twy;       R_(2, 1) = tyz + twx;       R_(2, 2) = 1 - (txx + tyy);
}

/* cu:329-415; JP is mdim x 6, JL is mdim x 3, both column-major with leading dimension mdim */
static void jacobians(const double* Xc, const double* q, const double* cam, int mdim, double* JP, double* JL)
{
	double R[9];
	quat_to_rot(q, R);
	const double X = Xc[0], Y = Xc[1], Z = Xc[2];
	const double invZ = 1 / Z;
	const double fu = cam[0], fv = cam[1], bf = cam[4];
#define JP_(i, j) JP[(j) * mdim + (i)]
#define JL_(i, j) JL[(j) * mdim + (i)]
	if (mdim == 2) {
		const double x = invZ * X, y = invZ * Y;
		const double fu_invZ = fu * invZ, fv_invZ = fv * invZ;
		for (int j = 0; j < 3; j++) {
			JL_(0, j) = -fu_invZ * (R_(0, j) - x * R_(2, j));
			JL_(1, j) = -fv_invZ * (R_(1, j) - y * R_(2, j));
		}
		JP_(0, 0) = +fu * x * y;       JP_(0, 1) = -fu * (1 + x * x); JP_(0, 2) = +fu * y;
		JP_(0, 3) = -fu_invZ;          JP_(0, 4) = 0;                 JP_(0, 5) = +fu_invZ * x;
		JP_(1, 0) = +fv * (1 + y * y); JP_(1, 1) = -fv * x * y;       JP_(1, 2) = -fv * x;
		JP_(1, 3) = 0;                 JP_(1, 4) = -fv_invZ;          JP_(1, 5) = +fv_invZ * y;
	} else {
		const double invZZ = invZ * invZ;
		for (int j = 0; j < 3; j++) {
			JL_(0, j) = -fu * R_(0, j) * invZ + fu * X * R_(2, j) * invZZ;
			JL_(1, j) = -fv * R_(1, j) * invZ + fv * Y * R_(2, j) * invZZ;
			JL_(2, j) = JL_(0, j) - bf * R_(2, j) * invZZ;
		}
		JP_(0, 0) = X * Y * invZZ * fu;         JP_(0, 1) = -(1 + (X * X * invZZ)) * fu; JP_(0, 2) = Y * invZ * fu;
		JP_(0, 3) = -1 * invZ * fu;             JP_(0, 4) = 0;                           JP_(0, 5) = X * invZZ * fu;
		JP_(1, 0) = (1 + Y * Y * invZZ) * fv;   JP_(1, 1) = -X * Y * invZZ * fv;         JP_(1, 2) = -X * invZ * fv;
		JP_(1, 3) = 0;                          JP_(1, 4) = -1 * invZ * fv;              JP_(1, 5) = Y * invZZ * fv;
		JP_(2, 0) = JP_(0, 0) - bf * Y * invZZ; JP_(2, 1) = JP_(0, 1) + bf * X * invZZ;  JP_(2, 2) = JP_(0, 2);
		JP_(2, 3) = JP_(0, 3);                  JP_(2, 4) = 0;                           JP_(2, 5) = JP_(0, 5) - bf * invZZ;
	}
#undef JP_
#undef JL_
}
#undef R_

/* cu:692-727 */
static double rk_rho(int type, double delta, double x)
{
	const double d2 = delta * delta;
	if (type == 1) return x <= d2 ? x : (2 * sqrt(x) * delta - d2);
	if (type == 2) {
		const double maxv = (1.0 / 3) * d2;
		const double u = 1 - x / d2;
		return x <= d2 ? maxv * (1 - u * u * u) : maxv;
	}
	return x;
}
static double rk_drho(int type, double delta, double x)
{
	const double d2 = delta * delta;
	if (type == 1) return x <= d2 ? 1 : (delta / sqrt(x));
	if (type == 2) { const double u = 1 - x / d2; return x <= d2 ? u * u : 0; }
	return 1;
}

/* cu:417-452, closed-form adjugate inverse of a symmetric 3x3 (column-major) */
static void sym3_inv(const double* A, double* B)
{
	const double A00 = A[0], A01 = A[3], A11 = A[4], A02 = A[2], A12 = A[7], A22 = A[8];
	const double det = A00 * A11 * A22 + A01 * A12 * A02 + A02 * A01 * A12
		- A00 * A12 * A12 - A02 * A11 * A02 - A01 * A01 * A22;
	const double id = 1 / det;
	const double B00 = id * (A11 * A22 - A12 * A12);
	const double B01 = id * (A02 * A12 - A01 * A22);
	const double B11 = id * (A00 * A22 - A02 * A02);
	const double B02 = id * (A01 * A12 - A02 * A11);
	const double B12 = id * (A02 * A01 - A00 * A12);
	const double B22 = id * (A00 * A11 - A01 * A01);
	B[0] = B00; B[3] = B01; B[6] = B02;
	B[1] = B01; B[4] = B11; B[7] = B12;
	B[2] = B02; B[5] = B12; B[8] = B22;
}

/* ---------------------------------------------------------------- structure */

static int cmp_int(const void* a, const void* b) { return *(const int*)a - *(const int*)b; }

/* Hpl CSC sorted by (iL, iP): cu:1158-1173 (thrust::sort LessColId + histogram + scan).
 * Ties (duplicate (P,L) pairs) are broken by edge id here; the reference leaves them unordered. */
static void build_hpl_structure(bao* h)
{
	const int E = h->E, numL = h->numL;
	h->edge2Hpl = (int*)malloc(sizeof(int) * (E > 0 ? E : 1));
	h->hplColPtr = (int*)calloc(numL + 1, sizeof(int));
	int n = 0;
	for (int e = 0; e < E; e++) {
		h->edge2Hpl[e] = -1;
		if (!h->flag[e]) { h->hplColPtr[h->ePL[2 * e + 1] + 1]++; n++; }
	}
	h->nhpl = n;
	for (int l = 0; l < numL; l++) h->hplColPtr[l + 1] += h->hplColPtr[l];
	h->hplRowInd = (int*)malloc(sizeof(int) * (n > 0 ? n : 1));
	h->hplEdge = (int*)malloc(sizeof(int) * (n > 0 ? n : 1));
	/* counting sort by iP first (stable), then bucket by iL -> sorted by (iL, iP, edge id) */
	int* cntP = (int*)calloc(h->numP + 1, sizeof(int));
	for (int e = 0; e < E; e++) if (!h->flag[e]) cntP[h->ePL[2 * e] + 1]++;
	for (int p = 0; p < h->numP; p++) cntP[p + 1] += cntP[p];
	int* byP = (int*)malloc(sizeof(int) * (n > 0 ? n : 1));
	for (int e = 0; e < E; e++) if (!h->flag[e]) byP[cntP[h->ePL[2 * e]]++] = e;
	int* fill = (int*)malloc(sizeof(int) * (numL + 1));
	memcpy(fill, h->hplColPtr, sizeof(int) * (numL + 1));
	for (int k = 0; k < n; k++) {
		const int e = byP[k];
		const int pos = fill[h->ePL[2 * e + 1]]++;
		h->hplRowInd[pos] = h->ePL[2 * e];
		h->hplEdge[pos] = e;
		h->edge2Hpl[e] = pos;
	}
	free(cntP); free(byP); free(fill);
}

/* First column partner of Hpl block i of landmark l: i, or -- when its pose observes l through more than one edge (a repeated
 * pair, which g2o sums and so does the engine; the reference pairs only i <= j and leaves Hsc(a,a) without W_j Hpl_i^T) -- the
 * first of that pose's blocks in the column (the column is sorted by pose). */
static int first_partner(const bao* h, int l, int i)
{
	int j = i;
	while (j > h->hplColPtr[l] && h->hplRowInd[j - 1] == h->hplRowInd[i]) j--;
	return j;
}

/* Upper-triangular BSR pattern of Hsc from landmark co-visibility:
 * sparse_block_matrix.cpp:55-133 (constructFromVertices), columns ascending per row. */
static void build_hsc_structure(bao* h)
{
	const int numP = h->numP, numL = h->numL;
	/* count products and collect (row,col) pairs */
	long nmul = 0;
	for (int l = 0; l < numL; l++)
		for (int i = h->hplColPtr[l]; i < h->hplColPtr[l + 1]; i++) nmul += h->hplColPtr[l + 1] - first_partner(h, l, i);
	h->nmul = (int)nmul;
	/* + one (p,p) key per free pose: the reference only gets a diagonal block when the pose has a
	 * free-free edge (and then mis-addresses Hpp otherwise, cu:955-962); we always keep the diagonal. */
	nmul += numP;
	int64_t* keys = (int64_t*)malloc(sizeof(int64_t) * (nmul > 0 ? nmul : 1));
	long m = 0;
	for (int p = 0; p < numP; p++) keys[m++] = ((int64_t)p << 32) | (uint32_t)p;
	for (int l = 0; l < numL; l++)
		for (int i = h->hplColPtr[l]; i < h->hplColPtr[l + 1]; i++)
			for (int j = first_partner(h, l, i); j < h->hplColPtr[l + 1]; j++)
				keys[m++] = ((int64_t)h->hplRowInd[i] << 32) | (uint32_t)h->hplRowInd[j];
	/* radix-free: sort 64-bit keys with two counting passes (col then row) */
	int64_t* tmp = (int64_t*)malloc(sizeof(int64_t) * (nmul > 0 ? nmul : 1));
	int* cnt = (int*)calloc(numP + 1, sizeof(int));
	for (long k = 0; k < nmul; k++) cnt[(int)(keys[k] & 0xffffffff) + 1]++;
	for (int p = 0; p < numP; p++) cnt[p + 1] += cnt[p];
	for (long k = 0; k < nmul; k++) tmp[cnt[(int)(keys[k] & 0xffffffff)]++] = keys[k];
	memset(cnt, 0, sizeof(int) * (numP + 1));
	for (long k = 0; k < nmul; k++) cnt[(int)(tmp[k] >> 32) + 1]++;
	for (int p = 0; p < numP; p++) cnt[p + 1] += cnt[p];
	for (long k = 0; k < nmul; k++) keys[cnt[(int)(tmp[k] >> 32)]++] = tmp[k];
	free(tmp); free(cnt);
	/* unique */
	h->hscRowPtr = (int*)calloc(numP + 1, sizeof(int));
	int nblk = 0;
	for (long k = 0; k < nmul; k++) if (k == 0 || keys[k] != keys[k - 1]) nblk++;
	h->nblk = nblk;
	h->hscColInd = (int*)malloc(sizeof(int) * (nblk > 0 ? nblk : 1));
	int b = 0;
	for (long k = 0; k < nmul; k++) {
		if (k == 0 || keys[k] != keys[k - 1]) {
			h->hscRowPtr[(int)(keys[k] >> 32) + 1]++;
			h->hscColInd[b++] = (int)(keys[k] & 0xffffffff);
		}
	}
	for (int p = 0; p < numP; p++) h->hscRowPtr[p + 1] += h->hscRowPtr[p];
	free(keys);
}

/* ---------------------------------------------------------------- block sparse Cholesky */

/* Exact minimum-degree ordering on the block graph with bitset adjacency; also yields the
 * filled column structures.  (Stands in for METIS ND + csrcholAnalysis, cuda_linear_solver.cpp:278-299,342-348;
 * the ordering does not change the mathematical solution.) */
static void chol_analyze(bao* h)
{
	const int n = h->numP;
	const int W = (n + 63) / 64;
	uint64_t* adj = (uint64_t*)calloc((size_t)n * W, sizeof(uint64_t));
	for (int r = 0; r < n; r++)
		for (int k = h->hscRowPtr[r]; k < h->hscRowPtr[r + 1]; k++) {
			const int c = h->hscColInd[k];
			if (c == r) continue;
			adj[(size_t)r * W + c / 64] |= 1ull << (c % 64);
			adj[(size_t)c * W + r / 64] |= 1ull << (r % 64);
		}
	int* deg = (int*)malloc(sizeof(int) * n);
	unsigned char* done = (unsigned char*)calloc(n, 1);
	for (int i = 0; i < n; i++) {
		int d = 0;
		for (int w = 0; w < W; w++) d += __builtin_popcountll(adj[(size_t)i * W + w]);
		deg[i] = d;
	}
	h->perm = (int*)malloc(sizeof(int) * n);
	h->iperm = (int*)malloc(sizeof(int) * n);
	h->Lptr = (int*)malloc(sizeof(int) * (n + 1));
	int** cols = (int**)malloc(sizeof(int*) * n);
	int* ncol = (int*)malloc(sizeof(int) * n);
	long total = 0;
	for (int k = 0; k < n; k++) {
		int best = -1;
		for (int i = 0; i < n; i++) if (!done[i] && (best < 0 || deg[i] < deg[best])) best = i;
		const int p = best;
		done[p] = 1; h->perm[k] = p; h->iperm[p] = k;
		uint64_t* ap = adj + (size_t)p * W;
		/* neighbours of p (all still uneliminated because eliminated nodes are removed below) */
		int cntn = 0;
		for (int w = 0; w < W; w++) cntn += __builtin_popcountll(ap[w]);
		cols[k] = (int*)malloc(sizeof(int) * (cntn + 1));
		ncol[k] = 0;
		for (int w = 0; w < W; w++) {
			uint64_t bits = ap[w];
			while (bits) { const int b = __builtin_ctzll(bits); bits &= bits - 1; cols[k][ncol[k]++] = w * 64 + b; }
		}
		/* make the neighbours a clique, remove p */
		for (int a = 0; a < ncol[k]; a++) {
			const int i = cols[k][a];
			uint64_t* ai = adj + (size_t)i * W;
			for (int w = 0; w < W; w++) ai[w] |= ap[w];
			ai[i / 64] &= ~(1ull << (i % 64));
			ai[p / 64] &= ~(1ull << (p % 64));
			int d = 0;
			for (int w = 0; w < W; w++) d += __builtin_popcountll(ai[w]);
			deg[i] = d;
		}
		total += ncol[k] + 1;
	}
	/* convert neighbour lists (original ids) to elimination positions, sorted, diagonal first */
	h->Lrow = (int*)malloc(sizeof(int) * total);
	h->Lval = (double*)malloc(sizeof(double) * 36 * total);
	int off = 0;
	for (int k = 0; k < n; k++) {
		h->Lptr[k] = off;
		h->Lrow[off++] = k;
		for (int a = 0; a < ncol[k]; a++) cols[k][a] = h->iperm[cols[k][a]];
		qsort(cols[k], ncol[k], sizeof(int), cmp_int);
		for (int a = 0; a < ncol[k]; a++) h->Lrow[off++] = cols[k][a];
		free(cols[k]);
	}
	h->Lptr[n] = off;
	h->posmap = (int*)malloc(sizeof(int) * n);
	free(cols); free(ncol); free(adj); free(deg); free(done);
	h->chol_ready = 1;
}

/* dense 6x6 Cholesky in place (lower, column-major); returns 0 on non-positive / tiny pivot
 * (cusolverSpDcsrcholZeroPivot with tol 1e-14, cuda_linear_solver.cpp:175-189) */
static int chol6(double* A)
{
	for (int j = 0; j < 6; j++) {
		double d = A[j * 6 + j];
		for (int k = 0; k < j; k++) d -= A[k * 6 + j] * A[k * 6 + j];
		if (!(d > 0)) return 0;
		d = sqrt(d);
		if (d < 1e-14) return 0;
		A[j * 6 + j] = d;
		for (int i = j + 1; i < 6; i++) {
			double s = A[j * 6 + i];
			for (int k = 0; k < j; k++) s -= A[k * 6 + i] * A[k * 6 + j];
			A[j * 6 + i] = s / d;
		}
	}
	for (int j = 1; j < 6; j++) for (int i = 0; i < j; i++) A[j * 6 + i] = 0;
	return 1;
}

/* B <- B * L^{-T}  (B 6x6 col-major, L lower) : solve X L^T = B */
static void trsm_right_lt(const double* L, double* B)
{
	for (int j = 0; j < 6; j++) {
		for (int k = 0; k < j; k++)
			for (int i = 0; i < 6; i++) B[j * 6 + i] -= B[k * 6 + i] * L[k * 6 + j];
		const double d = 1 / L[j * 6 + j];
		for (int i = 0; i < 6; i++) B[j * 6 + i] *= d;
	}
}

/* numeric factorisation A = L L^T on the filled block pattern, then solve.  Returns 0 on failure. */
static int chol_factor_solve(bao* h, const double* Hsc, const double* b, double* x)
{
	const int n = h->numP;
	if (!h->chol_ready) chol_analyze(h);
	const int total = h->Lptr[n];
	memset(h->Lval, 0, sizeof(double) * 36 * (size_t)total);
	/* scatter the upper BSR (block (r,c), r<=c, holds H(r,c)) into lower storage of the permuted matrix */
	for (int r = 0; r < n; r++) {
		for (int k = h->hscRowPtr[r]; k < h->hscRowPtr[r + 1]; k++) {
			const int c = h->hscColInd[k];
			const int pr = h->iperm[r], pc = h->iperm[c];
			const double* src = Hsc + 36 * (size_t)k;
			/* we need block (row=max, col=min) of the permuted matrix */
			const int col = pr < pc ? pr : pc, row = pr < pc ? pc : pr;
			int pos = -1;
			for (int a = h->Lptr[col]; a < h->Lptr[col + 1]; a++) if (h->Lrow[a] == row) { pos = a; break; }
			double* dst = h->Lval + 36 * (size_t)pos;
			/* src = H(r,c).  If (row,col) == (pr,pc) we need H(r,c); else H(c,r) = H(r,c)^T */
			if (row == pr && col == pc) { for (int e = 0; e < 36; e++) dst[e] = src[e]; }
			else { for (int j = 0; j < 6; j++) for (int i = 0; i < 6; i++) dst[j * 6 + i] = src[i * 6 + j]; }
		}
	}
	/* right-looking block Cholesky */
	for (int k = 0; k < n; k++) {
		const int c0 = h->Lptr[k], c1 = h->Lptr[k + 1];
		double* Lkk = h->Lval + 36 * (size_t)c0;
		if (!chol6(Lkk)) return 0;
		for (int a = c0 + 1; a < c1; a++) trsm_right_lt(Lkk, h->Lval + 36 * (size_t)a);
		for (int a = c0 + 1; a < c1; a++) {
			const int j = h->Lrow[a];            /* target column */
			const double* Ljk = h->Lval + 36 * (size_t)a;
			for (int s = h->Lptr[j]; s < h->Lptr[j + 1]; s++) h->posmap[h->Lrow[s]] = s;
			for (int bidx = a; bidx < c1; bidx++) {
				const int i = h->Lrow[bidx];
				const double* Lik = h->Lval + 36 * (size_t)bidx;
				double* T = h->Lval + 36 * (size_t)h->posmap[i];
				/* T(6x6) -= Lik * Ljk^T */
				for (int cc = 0; cc < 6; cc++)
					for (int m = 0; m < 6; m++) {
						const double v = Ljk[m * 6 + cc];
						for (int rr = 0; rr < 6; rr++) T[cc * 6 + rr] -= Lik[m * 6 + rr] * v;
					}
			}
		}
	}
	/* solve L y = P b ; L^T z = y ; x = P^T z */
	double* y = (double*)malloc(sizeof(double) * 6 * n);
	for (int k = 0; k < n; k++) for (int i = 0; i < 6; i++) y[6 * k + i] = b[6 * h->perm[k] + i];
	for (int k = 0; k < n; k++) {
		const int c0 = h->Lptr[k], c1 = h->Lptr[k + 1];
		const double* Lkk = h->Lval + 36 * (size_t)c0;
		double* yk = y + 6 * k;
		for (int j = 0; j < 6; j++) {
			yk[j] /= Lkk[j * 6 + j];
			for (int i = j + 1; i < 6; i++) yk[i] -= Lkk[j * 6 + i] * yk[j];
		}
		for (int a = c0 + 1; a < c1; a++) {
			const double* Lik = h->Lval + 36 * (size_t)a;
			double* yi = y + 6 * h->Lrow[a];
			for (int j = 0; j < 6; j++) for (int i = 0; i < 6; i++) yi[i] -= Lik[j * 6 + i] * yk[j];
		}
	}
	for (int k = n - 1; k >= 0; k--) {
		const int c0 = h->Lptr[k], c1 = h->Lptr[k + 1];
		const double* Lkk = h->Lval + 36 * (size_t)c0;
		double* yk = y + 6 * k;
		for (int a = c0 + 1; a < c1; a++) {
			const double* Lik = h->Lval + 36 * (size_t)a;
			const double* yi = y + 6 * h->Lrow[a];
			for (int j = 0; j < 6; j++) { double s = 0; for (int i = 0; i < 6; i++) s += Lik[j * 6 + i] * yi[i]; yk[j] -= s; }
		}
		for (int j = 5; j >= 0; j--) {
			for (int i = j + 1; i < 6; i++) yk[j] -= Lkk[j * 6 + i] * yk[i];
			yk[j] /= Lkk[j * 6 + j];
		}
	}
	for (int k = 0; k < n; k++) for (int i = 0; i < 6; i++) x[6 * h->perm[k] + i] = y[6 * k + i];
	free(y);
	return 1;
}

/* ---------------------------------------------------------------- create / destroy */

static double* dupd(const double* src, size_t n)
{
	double* p = (double*)malloc(sizeof(double) * (n > 0 ? n : 1));
	if (n) memcpy(p, src, sizeof(double) * n);
	return p;
}

bao* bao_create(const bao_problem* pr, const int rk_type[2], const double rk_delta[2])
{
	bao* h = (bao*)calloc(1, sizeof(bao));
	h->Pall = pr->Pall; h->numP = pr->numP; h->Lall = pr->Lall; h->numL = pr->numL;
	h->E2 = pr->E2; h->E3 = pr->E3; h->E = pr->E2 + pr->E3;
	for (int i = 0; i < 2; i++) { h->rk_type[i] = rk_type[i]; h->rk_delta[i] = rk_delta[i]; }
	h->q = dupd(pr->q, 4 * (size_t)h->Pall); h->t = dupd(pr->t, 3 * (size_t)h->Pall);
	h->cam = dupd(pr->cam, 5 * (size_t)h->Pall); h->Xw = dupd(pr->Xw, 3 * (size_t)h->Lall);
	h->q_bak = dupd(pr->q, 4 * (size_t)h->Pall); h->t_bak = dupd(pr->t, 3 * (size_t)h->Pall);
	h->Xw_bak = dupd(pr->Xw, 3 * (size_t)h->Lall);
	const int E = h->E;
	h->ePL = (int*)malloc(sizeof(int) * 2 * (E > 0 ? E : 1));
	h->meas = (double*)calloc(3 * (size_t)(E > 0 ? E : 1), sizeof(double));
	h->omega = (double*)malloc(sizeof(double) * (E > 0 ? E : 1));
	h->flag = (unsigned char*)malloc(E > 0 ? E : 1);
	h->err = (double*)calloc(3 * (size_t)(E > 0 ? E : 1), sizeof(double));
	h->Xc = (double*)calloc(3 * (size_t)(E > 0 ? E : 1), sizeof(double));
	for (int e = 0; e < h->E2; e++) {
		h->ePL[2 * e] = pr->idx2[2 * e]; h->ePL[2 * e + 1] = pr->idx2[2 * e + 1];
		h->meas[3 * e] = pr->meas2[2 * e]; h->meas[3 * e + 1] = pr->meas2[2 * e + 1];
		h->omega[e] = pr->omega2[e];
	}
	for (int k = 0; k < h->E3; k++) {
		const int e = h->E2 + k;
		h->ePL[2 * e] = pr->idx3[2 * k]; h->ePL[2 * e + 1] = pr->idx3[2 * k + 1];
		for (int i = 0; i < 3; i++) h->meas[3 * e + i] = pr->meas3[3 * k + i];
		h->omega[e] = pr->omega3[k];
	}
	for (int e = 0; e < E; e++)  /* cpp:566-572 makeEdgeFlag */
		h->flag[e] = (unsigned char)((h->ePL[2 * e] >= h->numP ? 2 : 0) | (h->ePL[2 * e + 1] >= h->numL ? 1 : 0));
	build_hpl_structure(h);
	build_hsc_structure(h);
	const int nP = h->numP > 0 ? h->numP : 1, nL = h->numL > 0 ? h->numL : 1;
	h->Hpp = (double*)calloc(36 * (size_t)nP, sizeof(double)); h->bp = (double*)calloc(6 * (size_t)nP, sizeof(double));
	h->Hll = (double*)calloc(9 * (size_t)nL, sizeof(double)); h->bl = (double*)calloc(3 * (size_t)nL, sizeof(double));
	h->Hpl = (double*)calloc(18 * (size_t)(h->nhpl > 0 ? h->nhpl : 1), sizeof(double));
	h->Hsc = (double*)calloc(36 * (size_t)(h->nblk > 0 ? h->nblk : 1), sizeof(double));
	h->bsc = (double*)calloc(6 * (size_t)nP, sizeof(double));
	h->invHll = (double*)calloc(9 * (size_t)nL, sizeof(double));
	h->xp = (double*)calloc(6 * (size_t)nP, sizeof(double)); h->xl = (double*)calloc(3 * (size_t)nL, sizeof(double));
	return h;
}

void bao_destroy(bao* h)
{
	if (!h) return;
	free(h->q); free(h->t); free(h->cam); free(h->Xw); free(h->q_bak); free(h->t_bak); free(h->Xw_bak);
	free(h->ePL); free(h->meas); free(h->omega); free(h->flag); free(h->err); free(h->Xc);
	free(h->hplColPtr); free(h->hplRowInd); free(h->edge2Hpl); free(h->hplEdge); free(h->hscRowPtr); free(h->hscColInd);
	free(h->Hpp); free(h->bp); free(h->Hll); free(h->bl); free(h->Hpl); free(h->Hsc); free(h->bsc); free(h->invHll);
	free(h->xp); free(h->xl);
	free(h->perm); free(h->iperm); free(h->Lptr); free(h->Lrow); free(h->Lval); free(h->posmap);
	free(h);
}

int bao_threads(void)
{
#ifdef _OPENMP
	return omp_get_max_threads();
#else
	return 1;
#endif
}

/* ---------------------------------------------------------------- LM stages */

/* cpp:368-382 + cu:732-786: residual = projection - measurement, Xc stored, sum of rho(omega*|e|^2) */
double bao_compute_errors(bao* h)
{
	double chi = 0;
#ifdef _OPENMP
#pragma omp parallel for reduction(+ : chi) schedule(static)
#endif
	for (int e = 0; e < h->E; e++) {
		const int mdim = e < h->E2 ? 2 : 3, ty = e < h->E2 ? 0 : 1;
		const int iP = h->ePL[2 * e], iL = h->ePL[2 * e + 1];
		double Xc[3], p[3], s = 0;
		project_w2c(h->q + 4 * iP, h->t + 3 * iP, h->Xw + 3 * iL, Xc);
		project_c2i(Xc, h->cam + 5 * iP, mdim, p);
		for (int i = 0; i < mdim; i++) { h->err[3 * e + i] = p[i] - h->meas[3 * e + i]; s += h->err[3 * e + i] * h->err[3 * e + i]; }
		for (int i = 0; i < 3; i++) h->Xc[3 * e + i] = Xc[i];
		chi += rk_rho(h->rk_type[ty], h->rk_delta[ty], h->omega[e] * s);
	}
	return chi;
}

/* cpp:384-410 + cu:788-839 (uses err/Xc of the preceding bao_compute_errors, like the reference) */
void bao_build_system(bao* h)
{
	memset(h->Hpp, 0, sizeof(double) * 36 * (size_t)h->numP); memset(h->bp, 0, sizeof(double) * 6 * (size_t)h->numP);
	memset(h->Hll, 0, sizeof(double) * 9 * (size_t)h->numL); memset(h->bl, 0, sizeof(double) * 3 * (size_t)h->numL);
	for (int e = 0; e < h->E; e++) {
		const int mdim = e < h->E2 ? 2 : 3, ty = e < h->E2 ? 0 : 1;
		const int iP = h->ePL[2 * e], iL = h->ePL[2 * e + 1], flag = h->flag[e];
		const double* r = h->err + 3 * e;
		double s = 0;
		for (int i = 0; i < mdim; i++) s += r[i] * r[i];
		const double w = h->omega[e] * rk_drho(h->rk_type[ty], h->rk_delta[ty], s * h->omega[e]);
		double JP[18], JL[9];
		jacobians(h->Xc + 3 * e, h->q + 4 * iP, h->cam + 5 * iP, mdim, JP, JL);
		if (!(flag & 2)) {
			double* H = h->Hpp + 36 * (size_t)iP; double* b = h->bp + 6 * (size_t)iP;
			for (int n = 0; n < 6; n++) for (int l = 0; l < 6; l++) {
				double d = 0; for (int m = 0; m < mdim; m++) d += JP[l * mdim + m] * JP[n * mdim + m];
				H[n * 6 + l] += w * d;
			}
			for (int l = 0; l < 6; l++) { double d = 0; for (int m = 0; m < mdim; m++) d += JP[l * mdim + m] * r[m]; b[l] += w * d; }
		}
		if (!(flag & 1)) {
			double* H = h->Hll + 9 * (size_t)iL; double* b = h->bl + 3 * (size_t)iL;
			for (int n = 0; n < 3; n++) for (int l = 0; l < 3; l++) {
				double d = 0; for (int m = 0; m < mdim; m++) d += JL[l * mdim + m] * JL[n * mdim + m];
				H[n * 3 + l] += w * d;
			}
			for (int l = 0; l < 3; l++) { double d = 0; for (int m = 0; m < mdim; m++) d += JL[l * mdim + m] * r[m]; b[l] += w * d; }
		}
		if (!flag) {
			double* H = h->Hpl + 18 * (size_t)h->edge2Hpl[e];
			for (int n = 0; n < 3; n++) for (int l = 0; l < 6; l++) {
				double d = 0; for (int m = 0; m < mdim; m++) d += JP[l * mdim + m] * JL[n * mdim + m];
				H[n * 6 + l] = w * d;
			}
		}
	}
}

/* cpp:412-418 + cu:877-904: max over the diagonals, starting from 0 */
double bao_max_diagonal(bao* h)
{
	double m = 0;
	for (int p = 0; p < h->numP; p++) for (int k = 0; k < 6; k++) m = fmax(m, h->Hpp[36 * (size_t)p + 7 * k]);
	for (int l = 0; l < h->numL; l++) for (int k = 0; k < 3; k++) m = fmax(m, h->Hll[9 * (size_t)l + 4 * k]);
	return m;
}

/* closed-form 6x6 solve by 3+3 Schur split: cu:617-664 */
static void solve_sym6(const double* H, const double* b, double* x)
{
	double Hpl[9], Hll[9], Hs[9], inv[9], W[9], bs[3], cl[3], invs[9];
	for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++) {
		Hpl[j * 3 + i] = H[(j + 3) * 6 + i]; Hll[j * 3 + i] = H[(j + 3) * 6 + i + 3]; Hs[j * 3 + i] = H[j * 6 + i];
	}
	sym3_inv(Hll, inv);
	for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++) { double s = 0; for (int k = 0; k < 3; k++) s += Hpl[k * 3 + i] * inv[j * 3 + k]; W[j * 3 + i] = s; }
	for (int j = 0; j < 3; j++) for (int i = 0; i < 3; i++) { double s = 0; for (int k = 0; k < 3; k++) s += W[k * 3 + i] * Hpl[k * 3 + j]; Hs[j * 3 + i] -= s; }
	for (int i = 0; i < 3; i++) { double s = 0; for (int k = 0; k < 3; k++) s += W[k * 3 + i] * b[3 + k]; bs[i] = b[i] - s; }
	sym3_inv(Hs, invs);
	for (int i = 0; i < 3; i++) { double s = 0; for (int k = 0; k < 3; k++) s += invs[k * 3 + i] * bs[k]; x[i] = s; }
	for (int i = 0; i < 3; i++) { double s = 0; for (int k = 0; k < 3; k++) s += Hpl[i * 3 + k] * x[k]; cl[i] = b[3 + i] - s; }
	for (int i = 0; i < 3; i++) { double s = 0; for (int k = 0; k < 3; k++) s += inv[k * 3 + i] * cl[k]; x[3 + i] = s; }
}

/* cpp:420-481: setLambda + solve (+ the caller restores nothing: lambda is applied on copies here) */
int bao_solve(bao* h, double lambda)
{
	const int numP = h->numP, numL = h->numL;
	if (numP > 0 && numL > 0) {
		/* cu:933-953 computeBschure */
		memcpy(h->bsc, h->bp, sizeof(double) * 6 * (size_t)numP);
		memset(h->Hsc, 0, sizeof(double) * 36 * (size_t)h->nblk);
		/* cu:955-962 initializeHschur: diagonal block is the first of each row */
		for (int p = 0; p < numP; p++) {
			double* D = h->Hsc + 36 * (size_t)h->hscRowPtr[p];
			memcpy(D, h->Hpp + 36 * (size_t)p, sizeof(double) * 36);
			for (int k = 0; k < 6; k++) D[7 * k] += lambda;
		}
		for (int l = 0; l < numL; l++) {
			double Hl[9], W[18];
			memcpy(Hl, h->Hll + 9 * (size_t)l, sizeof(Hl));
			for (int k = 0; k < 3; k++) Hl[4 * k] += lambda;
			double* inv = h->invHll + 9 * (size_t)l;
			sym3_inv(Hl, inv);
			const double* bl = h->bl + 3 * (size_t)l;
			for (int i = h->hplColPtr[l]; i < h->hplColPtr[l + 1]; i++) {
				const double* A = h->Hpl + 18 * (size_t)i;
				for (int c = 0; c < 3; c++) for (int r = 0; r < 6; r++) {
					double s = 0; for (int k = 0; k < 3; k++) s += A[k * 6 + r] * inv[c * 3 + k];
					W[c * 6 + r] = s;
				}
				const int rowi = h->hplRowInd[i];
				double* bs = h->bsc + 6 * (size_t)rowi;
				for (int r = 0; r < 6; r++) { double s = 0; for (int k = 0; k < 3; k++) s += W[k * 6 + r] * bl[k]; bs[r] -= s; }
				/* cu:964-1000: Hsc(row_i,row_j) -= W_i * Hpl_j^T for i <= j, and for j < i on the same pose (first_partner) */
				int k = h->hscRowPtr[rowi];
				for (int j = first_partner(h, l, i); j < h->hplColPtr[l + 1]; j++) {
					const int rowj = h->hplRowInd[j];
					while (h->hscColInd[k] < rowj) k++;
					const double* B = h->Hpl + 18 * (size_t)j;
					double* D = h->Hsc + 36 * (size_t)k;
					for (int c = 0; c < 6; c++) for (int r = 0; r < 6; r++) {
						double s = 0; for (int m = 0; m < 3; m++) s += W[m * 6 + r] * B[m * 6 + c];
						D[c * 6 + r] -= s;
					}
				}
			}
		}
		if (!chol_factor_solve(h, h->Hsc, h->bsc, h->xp)) return 0;
		/* cu:1029-1043 schurComplementPost */
		for (int l = 0; l < numL; l++) {
			double cl[3];
			for (int k = 0; k < 3; k++) cl[k] = h->bl[3 * (size_t)l + k];
			for (int i = h->hplColPtr[l]; i < h->hplColPtr[l + 1]; i++) {
				const double* A = h->Hpl + 18 * (size_t)i;
				const double* xp = h->xp + 6 * (size_t)h->hplRowInd[i];
				for (int c = 0; c < 3; c++) { double s = 0; for (int r = 0; r < 6; r++) s += A[c * 6 + r] * xp[r]; cl[c] -= s; }
			}
			const double* inv = h->invHll + 9 * (size_t)l;
			for (int r = 0; r < 3; r++) { double s = 0; for (int k = 0; k < 3; k++) s += inv[k * 3 + r] * cl[k]; h->xl[3 * (size_t)l + r] = s; }
		}
	} else if (numP > 0) {
		/* cu:1133-1140 pose-only */
		for (int p = 0; p < numP; p++) {
			double H[36]; memcpy(H, h->Hpp + 36 * (size_t)p, sizeof(H));
			for (int k = 0; k < 6; k++) H[7 * k] += lambda;
			solve_sym6(H, h->bp + 6 * (size_t)p, h->xp + 6 * (size_t)p);
		}
	} else {
		/* cu:1124-1131 landmark-only */
		for (int l = 0; l < numL; l++) {
			double H[9], inv[9]; memcpy(H, h->Hll + 9 * (size_t)l, sizeof(H));
			for (int k = 0; k < 3; k++) H[4 * k] += lambda;
			sym3_inv(H, inv);
			memcpy(h->invHll + 9 * (size_t)l, inv, sizeof(inv));
			const double* b = h->bl + 3 * (size_t)l;
			for (int r = 0; r < 3; r++) { double s = 0; for (int k = 0; k < 3; k++) s += inv[k * 3 + r] * b[k]; h->xl[3 * (size_t)l + r] = s; }
		}
	}
	return 1;
}

/* cu:492-521 (Eigen's algorithm), R column-major */
static void rot_to_quat(const double* R, double* q)
{
#define R_(i, j) R[(j) * 3 + (i)]
	double t = R_(0, 0) + R_(1, 1) + R_(2, 2);
	if (t > 0) {
		t = sqrt(t + 1);
		q[3] = 0.5 * t; t = 0.5 / t;
		q[0] = (R_(2, 1) - R_(1, 2)) * t; q[1] = (R_(0, 2) - R_(2, 0)) * t; q[2] = (R_(1, 0) - R_(0, 1)) * t;
	} else {
		int i = 0;
		if (R_(1, 1) > R_(0, 0)) i = 1;
		if (R_(2, 2) > R_(i, i)) i = 2;
		const int j = (i + 1) % 3, k = (j + 1) % 3;
		t = sqrt(R_(i, i) - R_(j, j) - R_(k, k) + 1);
		q[i] = 0.5 * t; t = 0.5 / t;
		q[3] = (R_(k, j) - R_(j, k)) * t; q[j] = (R_(j, i) + R_(i, j)) * t; q[k] = (R_(k, i) + R_(i, k)) * t;
	}
#undef R_
}

/* cu:551-592 updateExp + updatePose */
static void update_pose(const double* upd, double* q, double* t)
{
	const double wx = upd[0], wy = upd[1], wz = upd[2];
	const double theta = sqrt(wx * wx + wy * wy + wz * wz);
	/* skew1 / skew2, column-major (cu:454-473) */
	const double O1[9] = { 0, wz, -wy, -wz, 0, wx, wy, -wx, 0 };
	const double xx = wx * wx, yy = wy * wy, zz = wz * wz, xy = wx * wy, yz = wy * wz, zx = wz * wx;
	const double O2[9] = { -yy - zz, xy, zx, xy, -zz - xx, yz, zx, yz, -xx - yy };
	double a1, a2, a3, b2;
	if (theta < 0.00001) { a1 = 1.0; a2 = 0.5; b2 = 0.5; a3 = 1.0 / 6; }
	else {
		a1 = sin(theta) / theta; a2 = (1 - cos(theta)) / (theta * theta);
		b2 = a2; a3 = (theta - sin(theta)) / (theta * theta * theta);
	}
	double R[9], V[9];
	for (int k = 0; k < 9; k++) {
		const double I = (k == 0 || k == 4 || k == 8) ? 1.0 : 0.0;
		R[k] = I + a1 * O1[k] + a2 * O2[k];
		V[k] = I + b2 * O1[k] + a3 * O2[k];
	}
	double eq[4], et[3];
	rot_to_quat(R, eq);
	for (int i = 0; i < 3; i++) et[i] = V[0 * 3 + i] * upd[3] + V[1 * 3 + i] * upd[4] + V[2 * 3 + i] * upd[5];
	/* updatePose: t <- et + R(eq) t ; q <- normalize(eq * q) with w >= 0 */
	double u[3];
	rotate(eq, t, u);
	for (int i = 0; i < 3; i++) t[i] = et[i] + u[i];
	double r[4];
	r[3] = eq[3] * q[3] - eq[0] * q[0] - eq[1] * q[1] - eq[2] * q[2];
	r[0] = eq[3] * q[0] + eq[0] * q[3] + eq[1] * q[2] - eq[2] * q[1];
	r[1] = eq[3] * q[1] + eq[1] * q[3] + eq[2] * q[0] - eq[0] * q[2];
	r[2] = eq[3] * q[2] + eq[2] * q[3] + eq[0] * q[1] - eq[1] * q[0];
	double invn = 1 / sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3]);
	if (r[3] < 0) invn = -invn;
	for (int i = 0; i < 4; i++) q[i] = invn * r[i];
}

/* cpp:483-492 */
void bao_update(bao* h)
{
	for (int p = 0; p < h->numP; p++) update_pose(h->xp + 6 * (size_t)p, h->q + 4 * (size_t)p, h->t + 3 * (size_t)p);
	for (int l = 0; l < h->numL; l++) for (int k = 0; k < 3; k++) h->Xw[3 * (size_t)l + k] += h->xl[3 * (size_t)l + k];
}

/* cu:1070-1091: sum over [xp;xl] of x*(lambda*x + b) */
double bao_compute_scale(bao* h, double lambda)
{
	double s = 0;
	for (int i = 0; i < 6 * h->numP; i++) s += h->xp[i] * (lambda * h->xp[i] + h->bp[i]);
	for (int i = 0; i < 3 * h->numL; i++) s += h->xl[i] * (lambda * h->xl[i] + h->bl[i]);
	return s;
}

/* cu:841-875 non-robust omega*|e|^2 per edge */
void bao_chi_sqs(bao* h, double* out)
{
	for (int e = 0; e < h->E; e++) {
		const int mdim = e < h->E2 ? 2 : 3;
		const int iP = h->ePL[2 * e], iL = h->ePL[2 * e + 1];
		double Xc[3], p[3], s = 0;
		project_w2c(h->q + 4 * iP, h->t + 3 * iP, h->Xw + 3 * iL, Xc);
		project_c2i(Xc, h->cam + 5 * iP, mdim, p);
		for (int i = 0; i < mdim; i++) { const double d = p[i] - h->meas[3 * e + i]; s += d * d; }
		out[e] = h->omega[e] * s;
	}
}

static double clampd(double v, double lo, double hi) { return fmax(lo, fmin(v, hi)); }

/* cpp:793-857 */
int bao_optimize(bao* h, int niter, double* chi2_out, double* lambda_out, int* trials_out)
{
	const int maxq = 10;
	const double tau = 1e-5;
	double nu = 2, lambda = 0, F = 0;
	int nstat = 0;
	for (int it = 0; it < niter; it++) {
		F = bao_compute_errors(h);
		bao_build_system(h);
		if (it == 0) lambda = tau * bao_max_diagonal(h);
		int q = 0, ntrials = 0;
		double rho = -1;
		for (; q < maxq && rho < 0; q++) {
			ntrials++;
			memcpy(h->q_bak, h->q, sizeof(double) * 4 * (size_t)h->Pall);
			memcpy(h->t_bak, h->t, sizeof(double) * 3 * (size_t)h->Pall);
			memcpy(h->Xw_bak, h->Xw, sizeof(double) * 3 * (size_t)h->Lall);
			const int ok = bao_solve(h, lambda);
			bao_update(h);
			const double Fhat = bao_compute_errors(h);
			const double scale = bao_compute_scale(h, lambda) + 1e-3;
			rho = ok ? (F - Fhat) / scale : -1;
			if (rho > 0) {
				const double a = 2 * rho - 1;
				lambda *= clampd(1 - a * a * a, 1. / 3, 2. / 3);
				nu = 2; F = Fhat;
				break;
			} else {
				lambda *= nu; nu *= 2;
				memcpy(h->q, h->q_bak, sizeof(double) * 4 * (size_t)h->Pall);
				memcpy(h->t, h->t_bak, sizeof(double) * 3 * (size_t)h->Pall);
				memcpy(h->Xw, h->Xw_bak, sizeof(double) * 3 * (size_t)h->Lall);
			}
		}
		if (chi2_out) chi2_out[nstat] = F;
		if (lambda_out) lambda_out[nstat] = lambda;
		if (trials_out) trials_out[nstat] = ntrials;
		nstat++;
		if (q == maxq || rho <= 0 || !isfinite(lambda)) break;
	}
	return nstat;
}

/* ---------------------------------------------------------------- getters */
int bao_nhpl(const bao* h) { return h->nhpl; }
int bao_nblk(const bao* h) { return h->nblk; }
int bao_nmul(const bao* h) { return h->nmul; }

void bao_get_hpl_structure(const bao* h, int* colPtr, int* rowInd, int* edge2Hpl)
{
	if (colPtr) memcpy(colPtr, h->hplColPtr, sizeof(int) * (h->numL + 1));
	if (rowInd) memcpy(rowInd, h->hplRowInd, sizeof(int) * h->nhpl);
	if (edge2Hpl) memcpy(edge2Hpl, h->edge2Hpl, sizeof(int) * h->E);
}
void bao_get_hsc_structure(const bao* h, int* rowPtr, int* colInd)
{
	if (rowPtr) memcpy(rowPtr, h->hscRowPtr, sizeof(int) * (h->numP + 1));
	if (colInd) memcpy(colInd, h->hscColInd, sizeof(int) * h->nblk);
}
void bao_get_state(const bao* h, double* q, double* t, double* Xw)
{
	if (q) memcpy(q, h->q, sizeof(double) * 4 * (size_t)h->Pall);
	if (t) memcpy(t, h->t, sizeof(double) * 3 * (size_t)h->Pall);
	if (Xw) memcpy(Xw, h->Xw, sizeof(double) * 3 * (size_t)h->Lall);
}
void bao_set_state(bao* h, const double* q, const double* t, const double* Xw)
{
	if (q) memcpy(h->q, q, sizeof(double) * 4 * (size_t)h->Pall);
	if (t) memcpy(h->t, t, sizeof(double) * 3 * (size_t)h->Pall);
	if (Xw) memcpy(h->Xw, Xw, sizeof(double) * 3 * (size_t)h->Lall);
}
void bao_get_system(const bao* h, double* Hpp, double* bp, double* Hll, double* bl, double* Hpl)
{
	if (Hpp) memcpy(Hpp, h->Hpp, sizeof(double) * 36 * (size_t)h->numP);
	if (bp) memcpy(bp, h->bp, sizeof(double) * 6 * (size_t)h->numP);
	if (Hll) memcpy(Hll, h->Hll, sizeof(double) * 9 * (size_t)h->numL);
	if (bl) memcpy(bl, h->bl, sizeof(double) * 3 * (size_t)h->numL);
	if (Hpl) memcpy(Hpl, h->Hpl, sizeof(double) * 18 * (size_t)h->nhpl);
}
void bao_get_schur(const bao* h, double* Hsc, double* bsc, double* invHll)
{
	if (Hsc) memcpy(Hsc, h->Hsc, sizeof(double) * 36 * (size_t)h->nblk);
	if (bsc) memcpy(bsc, h->bsc, sizeof(double) * 6 * (size_t)h->numP);
	if (invHll) memcpy(invHll, h->invHll, sizeof(double) * 9 * (size_t)h->numL);
}
void bao_get_delta(const bao* h, double* xp, double* xl)
{
	if (xp) memcpy(xp, h->xp, sizeof(double) * 6 * (size_t)h->numP);
	if (xl) memcpy(xl, h->xl, sizeof(double) * 3 * (size_t)h->numL);
}
