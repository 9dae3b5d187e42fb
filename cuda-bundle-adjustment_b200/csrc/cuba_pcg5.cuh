// cuba_pcg5.cuh -- fifth-generation PCG on the reduced pose system: the two-level preconditioner of k_pcg4 inside the
// barrier-free exchange protocol of k_pcg3, with the block rows DISTRIBUTED OVER THE GPUs OF ONE NVLink DOMAIN.
//
//   mathematics   = k_pcg4: hat space A^ = L^-1 S L^-T, preconditioner M^-1 = I + Z^ (Z^T S Z)^-1 Z^^T (block-Jacobi + rigid-body
//                   coarse correction over pose aggregates), Chronopoulos-Gear single-reduction CG, stop on the block-Jacobi
//                   norm r^.r^ <= tol^2 r0^.r0^.  With A == 0 the coarse level is switched off (plain block-Jacobi = k_pcg3).
//   exchange      = k_pcg3: every value another CTA needs travels as "LL" words (fp64 split in two 32-bit halves, each next to
//                   a 32-bit tag in one 8-byte single-copy-atomic store); consumers poll, nobody fences, no grid barrier.
//   distribution  = the system's rows are cut into Gt = world * G contiguous ranges ("virtual CTAs"); GPU g runs the G CTAs
//                   [g*G, (g+1)*G) with their A^ blocks in registers / shared memory.  What crosses GPUs, per iteration:
//                     * the six w entries of the rows a peer's CTAs need (halo rows): the owner stores the same LL words into
//                       the peer's board through NVLink peer memory (cudaIpc-mapped), in the same instruction stream;
//                     * one rank summary (gamma, delta, rho and the restricted Z^^T w of the rank's aggregates): every CTA
//                       sums its GPU's partial board itself (one L2 hop, as k_pcg3), designated CTAs push the summary to every
//                       peer (one NVLink hop), everybody adds the summaries in rank order -> bit-identical scalars on all GPUs,
//                       hence identical iteration counts and exit passes without any host involvement.
//                   No NCCL call inside the solve.  world == 1 skips the rank hop.
//   coarse level  = c = (Z^T S Z)^-1 rc is computed ONCE per GPU and pass: every CTA holds the whole coarse residual rc (advanced by
//                   the CG recurrences from the published Z^^T w), multiplies it with ITS few rows of the explicit inverse (shared
//                   memory, fp32) and publishes the result on a third LL board; consumers poll the six entries of each aggregate
//                   their columns belong to.  One more L2 hop per pass, but the work is balanced: with k_pcg4's scheme (every CTA
//                   multiplies the rows of all its needed aggregates itself) the CTAs next to loop closures of the real ba_kitti_00
//                   needed 18 aggregates = 108 rows x 444 columns from L2 per pass and everybody waited for them (more than half of
//                   the cycles of a pass).
//   tags          = tagBase + pass, tagBase advanced by every solve (device-resident Pcg5Ctl): boards are never cleared;
//                   boards are double-buffered by pass parity and by solve parity (a peer may start the next solve while a
//                   slow CTA here still reads the last pass of this one).
// Replaces convertBSRToCSR + cuSOLVER csrchol (reference cuda_linear_solver.cpp:301-335) like the other PCG kernels.
#pragma once

#include "cuba_pcg4.cuh"

namespace cuba_b200 {

constexpr int PCG5_BLOCK = 256;
constexpr int PCG5_BPT = 2;                        // register-resident A^ blocks per thread
constexpr int PCG5_REGBLK = PCG5_BLOCK * PCG5_BPT;
constexpr int PCG5_CHUNK = PCG5_REGBLK;
constexpr int PCG5_REPL = 8;                       // replicas of the partial / summary boards
constexpr int PCG5_MAXWORLD = 8;
constexpr int PCG5_PCH = 8;                        // polled words in flight per thread
constexpr int PCG5_TPR = 16;                       // threads per row of the coarse slice product
constexpr int PCG5_MAXAGG = 148;                   // aggregates of a k_pcg5 plan (build_pcg5_plan's maxAgg) unless cfg.reserved[6] asks for fewer

// device-resident solve bookkeeping: read by every CTA at its start, changed only BETWEEN solves by k_pcg5_commit
struct Pcg5Ctl { unsigned int tagBase; unsigned int solve; int abort; int nbad; unsigned int advance; int pad[3]; };

struct Pcg5Dims {
	int capBlocks, needMax, maxRows, nc, maxNeedAgg, zhInSmem;
	int sliceRows; // rows of the inverse coarse matrix this CTA multiplies: ceil(nc / G)
	int npv;      // max(G * NP, world * NR): polled partial / summary words
	int nls;      // NR: words of a rank summary
};

// shared-memory carve-up, one definition for the host (size) and the device (pointers)
template <typename T>
struct Pcg5Layout {
	size_t blk, r, s, u, p, y, cc, rc, sc, c, zh, pv, ls, sq, ai, loc, rowPtr, woff, own, nagg, alist, diag, total;
	__host__ __device__ explicit Pcg5Layout(const Pcg5Dims& d)
	{
		size_t o = 0;
		auto take = [&o](size_t bytes, size_t align) { o = (o + align - 1) / align * align; const size_t at = o; o += bytes; return at; };
		blk = take((size_t)d.capBlocks * 36 * sizeof(T), 16);
		r = take((size_t)d.needMax * 6 * sizeof(T), 8);
		s = take((size_t)d.needMax * 6 * sizeof(T), 8);
		u = take((size_t)d.needMax * 6 * sizeof(T), 8);
		p = take((size_t)d.maxRows * 6 * sizeof(T), 8);
		y = take((size_t)d.maxRows * 6 * sizeof(T), 8);
		// block-product staging ([6][PCG5_CHUNK] T); between passes the polled w entries of the needed columns ([needMax][6] double),
		// so a dense row block (needMax > PCG5_CHUNK) widens it
		cc = take((size_t)(d.needMax > PCG5_CHUNK ? d.needMax : PCG5_CHUNK) * 6 * sizeof(double), 8);
		rc = take((size_t)d.nc * sizeof(T), 8);
		sc = take((size_t)d.nc * sizeof(T), 8);
		c = take((size_t)d.maxNeedAgg * 6 * sizeof(T), 8);
		zh = take(d.zhInSmem ? (size_t)d.needMax * 36 * sizeof(T) : 0, 8);
		pv = take((size_t)d.npv * sizeof(double), 8);
		ls = take((size_t)d.nls * sizeof(double), 8);
		sq = take((size_t)9 * d.maxRows * 6 * sizeof(double), 8);   // partial inner products of the (row, component) threads
		ai = take((size_t)d.sliceRows * d.nc * sizeof(float), 16);
		loc = take((size_t)d.capBlocks * sizeof(int), 4);
		rowPtr = take(((size_t)d.maxRows + 1) * sizeof(int), 4);
		woff = take((size_t)d.needMax * 6 * sizeof(int), 4);
		own = take((size_t)d.needMax * sizeof(int), 4);
		nagg = take((size_t)d.needMax * sizeof(int), 4);
		alist = take((size_t)d.maxNeedAgg * sizeof(int), 4);
		diag = take((size_t)d.maxRows * sizeof(int), 4);
		total = (o + 15) / 16 * 16;
	}
};

template <typename T>
struct Pcg5Args {
	const int* fRowPtr; const int* fColInd; const int* fLocal;   // symmetric-full BSR of the WHOLE system; fLocal per virtual CTA
	const T* fVal; T* fHat;
	const int* ctaRow;      // [Gt+1]
	const int* needPtr;     // [Gt+1]
	const int* needCol;
	int numP, G, rank, world;
	const T* Linv;          // [numP][36]   } k_pcg5_prep, every row on every rank
	const T* R0;            // [6 numP]     }
	const T* Zhat;          // [numP][36]   }
	const T* rc0;           // [nc]         }
	T* x;
	Pcg5Dims dims;
	int maxIters; double tol2;
	PcgStatus* status;
	// coarse level (A == 0: off)
	const float* AcInv; const int* naPtr; const int* naList; const int* needAgg;
	int A, gs;
	// boards of THIS GPU, [2 solve parity][2 pass parity]...
	unsigned long long* wBoard;      // ... [6 numP][2]
	unsigned long long* pBoard;      // ... [REPL][G * NP][2]
	unsigned long long* rBoard;      // ... [REPL][world * NR][2]
	unsigned long long* cBoard;      // ... [REPL][nc][2]   coarse correction c = Ac^-1 rc of the current pass
	unsigned long long* peerW[PCG5_MAXWORLD];   // the same boards of every rank (own entry = local pointer)
	unsigned long long* peerR[PCG5_MAXWORLD];
	Pcg5Ctl* peerCtl[PCG5_MAXWORLD];
	const unsigned char* rowPeers;   // [numP] bit r: rank r (not the owner) needs this row's w
	Pcg5Ctl* ctl;
	long long* timing;               // [G][8] per-phase clock64 sums (only with -DCUBA_PCG_TIMING)
};

// chol6_factor_and_inverse of cuba_pcg4.cuh with every loop unrolled: L and Li live in registers instead of local memory
// (k_pcg5_prep_rows spilled them with the rolled version).  Same operations
// in the same order.
template <typename T>
__device__ __forceinline__ bool chol6_factor_and_inverse_u(const T* A, T* L, T* Li)
{
#pragma unroll
	for (int i = 0; i < 36; i++) { L[i] = T(0); Li[i] = T(0); }
	bool ok = true;
#pragma unroll
	for (int j = 0; j < 6; j++) {
		T d = A[j * 6 + j];
#pragma unroll
		for (int k = 0; k < 6; k++) if (k < j) d -= L[k * 6 + j] * L[k * 6 + j];
		if (!(d > T(0))) ok = false;
		d = t_sqrt(ok ? d : T(1));
		L[j * 6 + j] = d;
		const T id = 1 / d;
#pragma unroll
		for (int i = 0; i < 6; i++) {
			if (i <= j) continue;
			T s = A[j * 6 + i];
#pragma unroll
			for (int k = 0; k < 6; k++) if (k < j) s -= L[k * 6 + i] * L[k * 6 + j];
			L[j * 6 + i] = s * id;
		}
	}
#pragma unroll
	for (int j = 0; j < 6; j++) {
		Li[j * 6 + j] = 1 / L[j * 6 + j];
#pragma unroll
		for (int i = 0; i < 6; i++) {
			if (i <= j) continue;
			T s = T(0);
#pragma unroll
			for (int k = 0; k < 6; k++) if (k >= j && k < i) s -= L[k * 6 + i] * Li[j * 6 + k];
			Li[j * 6 + i] = s / L[i * 6 + i];
		}
	}
	return ok;
}

// ---- preparation: factor every diagonal block, b^ = L^-1 b, Z^ = L^T Z, per-row share of rc0 = Z^^T b^ ----------------
template <typename T>
struct Pcg5PrepArgs {
	const int* fRowPtr; const int* fColInd; const T* fVal; const T* b; const T* Zx;
	int numP, A; const int* aggRow;
	int zhatFp32;   // 1: Z^ is rounded to fp32 before it is stored and used for rc0 (k_pcg5t keeps it in fp32 in shared memory)
	T* Linv; T* R0; T* Zhat; T* rcRow; T* rc0; Pcg5Ctl* ctl;
};

template <typename T>
__global__ void k_pcg5_prep_rows(const Pcg5PrepArgs<T> a)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.numP) return;
	// the diagonal block of row i: the columns of a row are ascending -> binary search (a linear walk is ~60 dependent loads)
	int d = -1;
	{
		int lo = a.fRowPtr[i], hi = a.fRowPtr[i + 1] - 1;
		while (lo < hi) { const int mid = (lo + hi) >> 1; if (a.fColInd[mid] < i) lo = mid + 1; else hi = mid; }
		if (lo <= hi && a.fColInd[lo] == i) d = lo;
	}
	T L[36], Li[36];
	T Ad[36];
#pragma unroll
	for (int e = 0; e < 36; e++) Ad[e] = d >= 0 ? a.fVal[36 * (size_t)d + e] : T(0);
	const bool ok = d >= 0 && chol6_factor_and_inverse_u(Ad, L, Li);
	if (!ok) {
		atomicAdd(&a.ctl->nbad, 1);
#pragma unroll
		for (int e = 0; e < 36; e++) { Li[e] = (e % 7) == 0 ? T(1) : T(0); L[e] = Li[e]; }
	}
#pragma unroll
	for (int e = 0; e < 36; e++) a.Linv[36 * (size_t)i + e] = Li[e];
	T bh[6], bi[6];
#pragma unroll
	for (int c = 0; c < 6; c++) bi[c] = a.b[6 * (size_t)i + c];
#pragma unroll
	for (int r = 0; r < 6; r++) {
		T s = T(0);
#pragma unroll
		for (int c = 0; c < 6; c++) if (c <= r) s += Li[c * 6 + r] * bi[c];
		bh[r] = s;
		a.R0[6 * (size_t)i + r] = s;
	}
	if (a.A > 0) {
		const T* Z = a.Zx + 36 * (size_t)i;
#pragma unroll
		for (int q = 0; q < 6; q++) {
			T zq[6];
#pragma unroll
			for (int k = 0; k < 6; k++) zq[k] = Z[q * 6 + k];
			T rcq = T(0);
#pragma unroll
			for (int r = 0; r < 6; r++) {
				T s = T(0);
#pragma unroll
				for (int k = 0; k < 6; k++) if (k >= r) s += L[r * 6 + k] * zq[k];       // Z^(r,q) = sum_{k>=r} L(k,r) Z(k,q)
				if (a.zhatFp32) s = (T)(float)s;
				a.Zhat[36 * (size_t)i + q * 6 + r] = s;
				rcq += s * bh[r];
			}
			a.rcRow[6 * (size_t)i + q] = rcq;
		}
	}
}
// rc0 of every aggregate: rows in ascending order (fixed order -> identical on every rank)
template <typename T>
__global__ void k_pcg5_prep_rc(const Pcg5PrepArgs<T> a)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= 6 * a.A) return;
	const int ag = e / 6, q = e - 6 * ag;
	T s = T(0);
	for (int i = a.aggRow[ag]; i < a.aggRow[ag + 1]; i++) s += a.rcRow[6 * (size_t)i + q];
	a.rc0[e] = s;
}

__device__ __forceinline__ void ll_load_raw(const unsigned long long* slot, unsigned long long& lo, unsigned long long& hi)
{
	asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(lo), "=l"(hi) : "l"(slot));
}
__device__ __forceinline__ bool ll_decode(unsigned long long lo, unsigned long long hi, unsigned int tag, double& v)
{
	if ((unsigned int)(lo >> 32) != tag || (unsigned int)(hi >> 32) != tag) return false;
	v = __longlong_as_double((long long)((lo & 0xffffffffull) | (hi << 32)));
	return true;
}

// Polls `n` LL words (slot of item i given by slotOf(i)) into dst[i]; PCG5_PCH loads of a thread are in flight together.
// Returns false when the solve was aborted (a peer vanished: spin limit).
template <typename SlotOf>
__device__ __forceinline__ bool ll_poll_many(int n, SlotOf slotOf, double* dst, unsigned int tag, Pcg5Ctl* ctl)
{
	const int tid = threadIdx.x;
	for (int base = 0; base < n; base += PCG5_BLOCK * PCG5_PCH) {
		unsigned int pend = 0;
#pragma unroll
		for (int u = 0; u < PCG5_PCH; u++) if (base + u * PCG5_BLOCK + tid < n) pend |= 1u << u;
		for (unsigned int spin = 0; pend; spin++) {
			unsigned long long lo[PCG5_PCH], hi[PCG5_PCH];
#pragma unroll
			for (int u = 0; u < PCG5_PCH; u++) if ((pend >> u) & 1u) ll_load_raw(slotOf(base + u * PCG5_BLOCK + tid), lo[u], hi[u]);
#pragma unroll
			for (int u = 0; u < PCG5_PCH; u++) if ((pend >> u) & 1u) {
				double v;
				if (ll_decode(lo[u], hi[u], tag, v)) { dst[base + u * PCG5_BLOCK + tid] = v; pend &= ~(1u << u); }
			}
			if ((spin & 1023u) == 1023u) {
				if (*(volatile int*)&ctl->abort) return false;
				if (spin >= PCG3_SPIN_LIMIT) { atomicExch(&ctl->abort, 1); return false; }
			}
		}
	}
	return true;
}

// BIG: the CTA may own more than 42 rows (up to 85): every thread then serves two (row, component) pairs in the row sums.
// lc: this CTA's index among the G CTAs of its rank (blockIdx.x in k_pcg5); the body reads neither blockIdx nor gridDim.
template <typename T, bool BIG>
__device__ __forceinline__ void pcg5_body(const Pcg5Args<T>& a, const int lc)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const Pcg5Layout<T> lay(a.dims);
	const int capBlocks = a.dims.capBlocks, nc = a.dims.nc;
	T* s_blk = reinterpret_cast<T*>(smem_raw + lay.blk);            // [36][capBlocks] blocks past the registers, element-major
	T* s_r = reinterpret_cast<T*>(smem_raw + lay.r);                // [needMax][6] residual of the needed columns
	T* s_s = reinterpret_cast<T*>(smem_raw + lay.s);                // [needMax][6] s = w + beta s
	T* s_u = reinterpret_cast<T*>(smem_raw + lay.u);                // [needMax][6] u = M^-1 r
	T* s_p = reinterpret_cast<T*>(smem_raw + lay.p);                // [maxRows][6]
	T* s_y = reinterpret_cast<T*>(smem_raw + lay.y);                // [maxRows][6]
	T* s_cc = reinterpret_cast<T*>(smem_raw + lay.cc);              // [6][PCG5_CHUNK] block products, component-major
	double* s_w = reinterpret_cast<double*>(smem_raw + lay.cc);     // polled w entries of the needed columns (same storage, other phase)
	T* s_rc = reinterpret_cast<T*>(smem_raw + lay.rc);              // [nc] coarse residual Z^^T r
	T* s_sc = reinterpret_cast<T*>(smem_raw + lay.sc);              // [nc]
	T* s_c = reinterpret_cast<T*>(smem_raw + lay.c);                // [maxNeedAgg][6]
	T* s_zh = reinterpret_cast<T*>(smem_raw + lay.zh);              // [needMax][36]
	double* s_pv = reinterpret_cast<double*>(smem_raw + lay.pv);    // polled partials, later polled rank summaries
	double* s_ls = reinterpret_cast<double*>(smem_raw + lay.ls);    // [NR] this rank's summary
	float* s_ai = reinterpret_cast<float*>(smem_raw + lay.ai);      // [nagg*6][nc] slices of AcInv
	int* s_loc = reinterpret_cast<int*>(smem_raw + lay.loc);
	int* s_rowPtr = reinterpret_cast<int*>(smem_raw + lay.rowPtr);
	int* s_woff = reinterpret_cast<int*>(smem_raw + lay.woff);      // [needMax*6] board offset of every needed w entry
	int* s_own = reinterpret_cast<int*>(smem_raw + lay.own);
	int* s_nagg = reinterpret_cast<int*>(smem_raw + lay.nagg);
	int* s_alist = reinterpret_cast<int*>(smem_raw + lay.alist);
	int* s_diag = reinterpret_cast<int*>(smem_raw + lay.diag);
	__shared__ int s_abort;

	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	const int G = a.G, cta = a.rank * G + lc, world = a.world;
	const bool coarse = a.A > 0;
	const int Aloc = coarse ? G / a.gs : 0;             // aggregates hosted by one rank (gs divides G)
	const int NP = coarse ? 9 : 3, NR = 3 + 6 * Aloc;
	const int row0 = a.ctaRow[cta], row1 = a.ctaRow[cta + 1], nrows = row1 - row0;
	const int need0 = a.needPtr[cta], nneed = a.needPtr[cta + 1] - need0;
	const int blk0 = a.fRowPtr[row0], nblkCta = a.fRowPtr[row1] - blk0;
	// BIG: no register-resident blocks -- the registers go to the loads in flight of the streamed part (see the product loop)
	constexpr int REGBLK = BIG ? 0 : PCG5_REGBLK;
	const int ncached = nblkCta > REGBLK ? (nblkCta - REGBLK < capBlocks ? nblkCta - REGBLK : capBlocks) : 0;
	const size_t n6 = 6 * (size_t)a.numP;
	const int nover = nblkCta - REGBLK - ncached > 0 ? nblkCta - REGBLK - ncached : 0;   // blocks read from the global copy every pass
	const size_t overBase = 36 * (size_t)(blk0 + REGBLK + ncached);
	int nagg = 0;
	// tags and the solve half of the boards
	const unsigned int tagBase = a.ctl->tagBase, half = a.ctl->solve & 1u;
	const int nbad = a.ctl->nbad;
	const size_t wStride = n6, pStride = (size_t)PCG5_REPL * G * NP, rStride = (size_t)PCG5_REPL * world * NR;   // words (16 B) per parity
	const size_t cStride = (size_t)PCG5_REPL * nc;
	const size_t wHalf = 2 * (size_t)half * wStride, pHalf = 2 * (size_t)half * pStride, rHalf = 2 * (size_t)half * rStride, cHalf = 2 * (size_t)half * cStride;
	const int srow0 = lc * a.dims.sliceRows, srow1 = srow0 + a.dims.sliceRows < nc ? srow0 + a.dims.sliceRows : nc;   // own rows of Ac^-1
	const int rep = lc % PCG5_REPL;

	if (tid == 0) s_abort = 0;
	for (int i = tid; i <= nrows; i += PCG5_BLOCK) s_rowPtr[i] = a.fRowPtr[row0 + i] - blk0;
	for (int i = tid; i < nneed; i += PCG5_BLOCK) {
		const int j = a.needCol[need0 + i];
		s_own[i] = (j >= row0 && j < row1) ? j - row0 : -1;
		if (coarse) s_nagg[i] = a.needAgg[need0 + i];
	}
	for (int i = tid; i < nneed * 6; i += PCG5_BLOCK) s_woff[i] = 6 * a.needCol[need0 + i / 6] + (i % 6);
	if (coarse) {
		const int na0 = a.naPtr[cta];
		nagg = a.naPtr[cta + 1] - na0;
		for (int i = tid; i < nagg; i += PCG5_BLOCK) s_alist[i] = a.naList[na0 + i];
		for (int i = tid; i < nc; i += PCG5_BLOCK) { s_rc[i] = a.rc0[i]; s_sc[i] = T(0); }
	}
	for (int i = tid; i < nrows * 6; i += PCG5_BLOCK) { s_p[i] = T(0); s_y[i] = T(0); }
	__syncthreads();
	for (int i = tid; i < nneed; i += PCG5_BLOCK) if (s_own[i] >= 0) s_diag[s_own[i]] = i;
	if (coarse) {
		if (a.dims.zhInSmem)
			for (int wi = tid; wi < nneed * 36; wi += PCG5_BLOCK) s_zh[wi] = __ldcg(a.Zhat + 36 * (size_t)a.needCol[need0 + wi / 36] + (wi % 36));
		for (int wi = tid; wi < (srow1 - srow0) * nc; wi += PCG5_BLOCK) s_ai[wi] = __ldg(a.AcInv + (size_t)srow0 * nc + wi);
	}

	// ---- A^_ij = L_i^-1 S_ij L_j^-T for the own rows: the first PCG5_REGBLK blocks stay in REGISTERS for the whole solve
	//      (thread n % BLOCK, slot n / BLOCK), later ones in shared memory (element-major), the rest in the global copy ----
	T breg[PCG5_BPT][36];
	int myLoc[PCG5_BPT];
#pragma unroll
	for (int u = 0; u < PCG5_BPT; u++) {
		myLoc[u] = -1;
#pragma unroll
		for (int e = 0; e < 36; e++) breg[u][e] = T(0);
	}
	{
		auto transform = [&](int n, T* out) {
			const int g = blk0 + n;
			int lo = 0, hi = nrows - 1;
			while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (s_rowPtr[mid] <= n) lo = mid; else hi = mid - 1; }
			const int i = row0 + lo, j = a.fColInd[g];
			const T* B = a.fVal + 36 * (size_t)g;
			const T* Li = a.Linv + 36 * (size_t)i;
			const T* Lj = a.Linv + 36 * (size_t)j;
			T tmp[36];
			for (int c = 0; c < 6; c++)
				for (int r = 0; r < 6; r++) {
					T s = T(0);
					for (int k = 0; k <= r; k++) s += Li[k * 6 + r] * B[c * 6 + k];
					tmp[c * 6 + r] = s;
				}
			for (int c = 0; c < 6; c++)
				for (int r = 0; r < 6; r++) {
					T s = T(0);
					for (int k = 0; k <= c; k++) s += tmp[k * 6 + r] * Lj[k * 6 + c];
					out[c * 6 + r] = s;
				}
		};
#pragma unroll
		for (int u = 0; u < PCG5_BPT; u++) {
			const int n = u * PCG5_BLOCK + tid;
			if (!BIG && n < nblkCta) {
				T out[36];
				transform(n, out);
#pragma unroll
				for (int e = 0; e < 36; e++) breg[u][e] = out[e];
				myLoc[u] = a.fLocal[blk0 + n];
			}
		}
		for (int n = REGBLK + tid; n < nblkCta; n += PCG5_BLOCK) {
			T out[36];
			transform(n, out);
			const int m = n - REGBLK;
			if (m < ncached) {
				for (int e = 0; e < 36; e++) s_blk[(size_t)e * capBlocks + m] = out[e];
				s_loc[m] = a.fLocal[blk0 + n];
			} else {
				// past the shared-memory cache: the global copy.  BIG: block-major (a thread streams its 288 contiguous bytes with
				// eighteen 16-byte loads in flight); else element-major inside this CTA's slice (coalesced 8-byte loads)
				if (BIG) { for (int e = 0; e < 36; e++) a.fHat[36 * (size_t)(blk0 + n) + e] = out[e]; }
				else { for (int e = 0; e < 36; e++) a.fHat[overBase + (size_t)e * nover + (m - ncached)] = out[e]; }
			}
		}
	}
	for (int wi = tid; wi < nneed * 6; wi += PCG5_BLOCK) {
		s_r[wi] = a.R0[s_woff[wi]];
		s_s[wi] = T(0);
		s_u[wi] = T(0);
	}
	__syncthreads();

	int status = 1, it = 0, kExit = 0;
	double gamma = 0, rho0 = 0, rho = 0, alpha = 0, beta = 0;
#ifdef CUBA_PCG_TIMING
	long long tacc[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
#endif
	int tpp = 1;                                         // threads per (row, component) pair of the row sums, a power of two
	while (tpp < 8 && nrows * 6 * tpp * 2 <= PCG5_BLOCK) tpp *= 2;
	if (nbad > 0) status = 2;
	else {
		// pass k = -1: u0 = M^-1 r0, w0 = A^ u0, first partials; pass k >= 0: CG iteration k.
		// Values published at the end of pass k-1 carry the tag tagBase + k + 1 and live in parity (k+1)&1.
		for (int k = -1;; k++) {
			kExit = k;
			if (k >= 0) {
				const unsigned int tag = tagBase + (unsigned int)(k + 1);
				const int par = (k + 1) & 1;
				PCG_T(t0);
				// ---- poll: w of the needed columns and this GPU's partial board (replica lc % REPL) ----
				{
					const int nW = nneed * 6, nPl = G * NP;
					const unsigned long long* wB = a.wBoard + 2 * (wHalf + (size_t)par * wStride);
					const unsigned long long* pB = a.pBoard + 2 * (pHalf + (size_t)par * pStride + (size_t)rep * nPl);
					// one destination array: s_w directly followed (logically) by s_pv -> two calls keep the indexing simple
					bool ok = ll_poll_many(nW, [&](int i) { return wB + 2 * (size_t)s_woff[i]; }, s_w, tag, a.ctl);
					ok = ok && ll_poll_many(nPl, [&](int i) { return pB + 2 * (size_t)i; }, s_pv, tag, a.ctl);
					if (!ok) s_abort = 1;
				}
				__syncthreads();
				PCG_T(t1);
				if (s_abort) { status = 3; break; }
				double gnew, delta, rnew;
				if (world == 1) {
					// ---- one GPU: every warp adds the three scalars over the CTAs itself (same order everywhere), no barrier;
					//      the restricted Z^^T w of an aggregate is summed by the thread that advances that coarse entry ----
					double v0 = 0, v1 = 0, v2 = 0;
					for (int c = lane; c < G; c += 32) { v0 += s_pv[c * NP]; v1 += s_pv[c * NP + 1]; v2 += s_pv[c * NP + 2]; }
					gnew = warp_sum(v0); delta = warp_sum(v1); rnew = warp_sum(v2);
				} else {
				// ---- this GPU's summary: gamma, delta, rho over its CTAs (one warp each), Z^^T w per local aggregate ----
				if (wid < 3) {
					double v = 0;
					for (int c = lane; c < G; c += 32) v += s_pv[c * NP + wid];
					v = warp_sum(v);
					if (lane == 0) s_ls[wid] = v;
				}
				if (coarse)
					for (int q = tid; q < 6 * Aloc; q += PCG5_BLOCK) {
						const int al = q / 6, comp = q - 6 * al;
						double v = 0;
						for (int c = al * a.gs; c < (al + 1) * a.gs; c++) v += s_pv[c * NP + 3 + comp];
						s_ls[3 + q] = v;
					}
				__syncthreads();
				{
					// ---- rank hop: designated CTAs push the summary to every rank's board (replica by replica), everybody polls ----
					const size_t rOff = rHalf + (size_t)par * rStride;
					for (int pr = lc; pr < world * PCG5_REPL; pr += G) {
						const int peer = pr / PCG5_REPL, rp = pr - peer * PCG5_REPL;
						unsigned long long* dst = a.peerR[peer] + 2 * (rOff + ((size_t)rp * world + a.rank) * NR);
						for (int q = tid; q < NR; q += PCG5_BLOCK) ll_store(dst + 2 * (size_t)q, s_ls[q], tag);
					}
					const unsigned long long* rB = a.rBoard + 2 * (rOff + (size_t)rep * world * NR);
					const bool ok = ll_poll_many(world * NR, [&](int i) { return rB + 2 * (size_t)i; }, s_pv, tag, a.ctl);
					if (!ok) s_abort = 1;
					__syncthreads();
					if (s_abort) { status = 3; break; }
					gnew = 0; delta = 0; rnew = 0;
					for (int r = 0; r < world; r++) { gnew += s_pv[r * NR]; delta += s_pv[r * NR + 1]; rnew += s_pv[r * NR + 2]; }
				}
				}
				PCG_T(t2);
				if (!(gnew == gnew) || !(delta == delta) || !(rnew == rnew)) { status = 2; break; }
				if (k == 0) {
					gamma = gnew; rho0 = rho = rnew;
					if (rho0 <= 0) { status = 0; break; }
					if (!(delta > 0) || !(gamma > 0)) { status = 2; break; }
					alpha = gamma / delta; beta = 0;
				} else {
					it = k;
					rho = rnew;
					if (rnew <= a.tol2 * rho0) { status = 0; break; }       // the block-Jacobi norm r' D^-1 r, as in k_pcg2/3/4
					if (!(gnew > 0)) { status = 2; break; }
					beta = gnew / gamma;
					const double ga = gamma * alpha;
					const double den = delta * ga - gnew * gnew;          // = ga (delta - beta g'/alpha)
					if (!(den > 0) || !(ga > 0)) { gamma = gnew; status = 2; break; }
					alpha = gnew * ga / den;
					gamma = gnew;
				}
				if (k >= a.maxIters) { status = 1; break; }
				// ---- advance s, r (needed columns), p, y (own rows; u_k is still in s_u) and the coarse residual ----
				for (int wi = tid; wi < nneed * 6; wi += PCG5_BLOCK) {
					const T snew = (T)s_w[wi] + (T)beta * s_s[wi];
					const T rold = s_r[wi];
					s_s[wi] = snew;
					s_r[wi] = rold - (T)alpha * snew;
					const int own = s_own[wi / 6];
					if (own >= 0) {
						const int o = own * 6 + (wi % 6);
						const T p = (coarse ? s_u[wi] : rold) + (T)beta * s_p[o];
						s_p[o] = p;
						s_y[o] += (T)alpha * p;
					}
				}
				if (coarse)
					for (int q = tid; q < nc; q += PCG5_BLOCK) {
						// global aggregate q/6 = rank r, local aggregate al
						double wcv;
						if (world > 1) wcv = s_pv[(q / (6 * Aloc)) * NR + 3 + (q % (6 * Aloc))];
						else {
							const int al = q / 6, comp = q - 6 * al;
							wcv = 0;
							for (int c = al * a.gs; c < (al + 1) * a.gs; c++) wcv += s_pv[c * NP + 3 + comp];
						}
						const T sc = (T)wcv + (T)beta * s_sc[q];
						s_sc[q] = sc;
						s_rc[q] -= (T)alpha * sc;
					}
				__syncthreads();
				PCG_T(t3);
				PCG_ACC(0, t0, t1); PCG_ACC(1, t1, t2); PCG_ACC(2, t2, t3);
			}
			PCG_T(t4);
			const T* s_v = s_r;                                   // the vector A^ is applied to
			if (coarse) {
				// ---- c = Ac^-1 rc: this CTA's rows (one warp per row, fixed-order butterfly), published for the whole GPU ----
				const unsigned int ctag = tagBase + (unsigned int)(k + 2);
				const int cpar = (k + 2) & 1;
				unsigned long long* cB = a.cBoard + 2 * (cHalf + (size_t)cpar * cStride);
				for (int rowi = srow0 + wid; rowi < srow1; rowi += PCG5_BLOCK / 32) {
					const float* Arow = s_ai + (size_t)(rowi - srow0) * nc;
					T sacc = T(0);
					for (int q = lane; q < nc; q += 32) sacc += (T)Arow[q] * s_rc[q];
					sacc = warp_sum(sacc);
					if (lane < PCG5_REPL) ll_store(cB + 2 * ((size_t)lane * nc + rowi), (double)sacc, ctag);
				}
				{
					const unsigned long long* cR = cB + 2 * ((size_t)rep * nc);
					double* cdst = sizeof(T) == 8 ? reinterpret_cast<double*>(s_c) : s_pv;
					const bool ok = ll_poll_many(nagg * 6, [&](int i) { return cR + 2 * (size_t)(s_alist[i / 6] * 6 + (i % 6)); }, cdst, ctag, a.ctl);
					if (!ok) s_abort = 1;
				}
				__syncthreads();
				if (s_abort) { status = 3; break; }
				if (sizeof(T) != 8) {
					for (int i = tid; i < nagg * 6; i += PCG5_BLOCK) s_c[i] = (T)s_pv[i];
					__syncthreads();
				}
				// ---- u_j = r_j + Z^_j c_a(j) for every needed column ----
				for (int wi = tid; wi < nneed * 6; wi += PCG5_BLOCK) {
					const int c = wi / 6, comp = wi - 6 * c;
					const T* cc = s_c + 6 * (size_t)s_nagg[c];
					T u = s_r[wi];
					if (a.dims.zhInSmem) {
						const T* Zh = s_zh + 36 * (size_t)c + comp;
#pragma unroll
						for (int q = 0; q < 6; q++) u += Zh[6 * q] * cc[q];
					} else {
						const T* Zh = a.Zhat + 36 * (size_t)(s_woff[wi] / 6) + comp;
#pragma unroll
						for (int q = 0; q < 6; q++) u += __ldcg(Zh + 6 * q) * cc[q];
					}
					s_u[wi] = u;
				}
				__syncthreads();
				s_v = s_u;
			}
			PCG_T(t5);
			// ---- w_{k+1} = A^ u_{k+1} for the own rows: block products from registers, then per-row sums ----
			const unsigned int otag = tagBase + (unsigned int)(k + 2);
			const int opar = (k + 2) & 1;
			// (row, component) pairs of this thread: pair tid / tpp, and -- only when the CTA owns more than 42 rows (tpp == 1) -- pair tid + BLOCK
			constexpr int NPU = BIG ? 2 : 1;
			T wacc[NPU];
#pragma unroll
			for (int pu = 0; pu < NPU; pu++) wacc[pu] = T(0);
			const int npairs = nrows * 6;
			for (int cs = 0; cs < nblkCta; cs += PCG5_CHUNK) {
				if (cs > 0) __syncthreads();
#pragma unroll
				for (int u = 0; u < PCG5_BPT; u++) {
					const int n = cs + u * PCG5_BLOCK + tid;
					T y[6] = { T(0), T(0), T(0), T(0), T(0), T(0) };
					if (!BIG && cs == 0) {
						if (myLoc[u] >= 0) {
							const T* rj = s_v + 6 * (size_t)myLoc[u];
#pragma unroll
							for (int c = 0; c < 6; c++) {
								const T rc = rj[c];
#pragma unroll
								for (int r = 0; r < 6; r++) y[r] += breg[u][c * 6 + r] * rc;
							}
						}
					} else if (n < nblkCta) {
						const int m = n - REGBLK;
						const bool cached = m < ncached;
						const int loc = cached ? s_loc[m] : a.fLocal[blk0 + n];
						if (loc >= 0) {
							const T* rj = s_v + 6 * (size_t)loc;
							if (cached) {
								const T* B = s_blk + m;
								const size_t st = (size_t)capBlocks;
#pragma unroll
								for (int c = 0; c < 6; c++) {
									const T rc = rj[c];
#pragma unroll
									for (int r = 0; r < 6; r++) y[r] += B[(c * 6 + r) * st] * rc;
								}
							} else if (BIG) {
								// streamed block: all 288 bytes requested before the first use (measured: requesting the blocks of both
								// chunk slots at once, 144 registers of loads in flight, is slower -- spills and L1 thrash)
								const T* B = a.fHat + 36 * (size_t)(blk0 + n);
								T bv[36];
#pragma unroll
								for (int x = 0; x < 36; x += 2) {      // plain (coherent) vector loads: this CTA wrote the block earlier in this launch
									const typename V2<T>::type v2 = *reinterpret_cast<const typename V2<T>::type*>(B + x);
									bv[x] = v2.x; bv[x + 1] = v2.y;
								}
#pragma unroll
								for (int c = 0; c < 6; c++) {
									const T rc = rj[c];
#pragma unroll
									for (int r = 0; r < 6; r++) y[r] += bv[c * 6 + r] * rc;
								}
							} else {
								const T* B = a.fHat + overBase + (m - ncached);
#pragma unroll 1
								for (int c = 0; c < 6; c++) {
									const T rc = rj[c];
#pragma unroll
									for (int r = 0; r < 6; r++) { y[r] += __ldcg(B) * rc; B += nover; }
								}
							}
						}
					}
#pragma unroll
					for (int r = 0; r < 6; r++) s_cc[r * PCG5_CHUNK + u * PCG5_BLOCK + tid] = y[r];
				}
				__syncthreads();
#pragma unroll
				for (int pu = 0; pu < NPU; pu++) {
					const int pair = tid / tpp + pu * PCG5_BLOCK, sub = tid % tpp;
					if (pair < npairs && (pu == 0 || tpp == 1)) {       // nrows * 6 <= 2 * PCG5_BLOCK (checked on the host)
						const int li = pair / 6, comp = pair - 6 * li;
						int n0 = s_rowPtr[li], n1 = s_rowPtr[li + 1];
						n0 = (n0 > cs ? n0 : cs) - cs;
						n1 = (n1 < cs + PCG5_CHUNK ? n1 : cs + PCG5_CHUNK) - cs;
						T s0 = T(0), s1 = T(0);
						const T* col = s_cc + comp * PCG5_CHUNK;
						int q = n0 + sub;
						for (; q + tpp < n1; q += 2 * tpp) { s0 += col[q]; s1 += col[q + tpp]; }
						if (q < n1) s0 += col[q];
						wacc[pu] += s0 + s1;
					}
				}
			}
			for (int o = 1; o < tpp; o <<= 1) wacc[0] += __shfl_xor_sync(0xffffffffu, wacc[0], o);
			PCG_T(t6);
			// ---- publish w (own board + the boards of the ranks that need the row), partial inner products, Z^^T w ----
			// The nine quantities of the (row, component) threads go to shared memory; afterwards warp w adds quantity w (warp 0
			// also the ninth) in a fixed order and its first REPL lanes publish the replicas.
			const int nact = nrows * 6;                           // active threads: tid = pair * tpp
			double* s_q = reinterpret_cast<double*>(smem_raw + lay.sq);   // [9][nact]; read below, rewritten only after the next pass's barriers
#pragma unroll
			for (int pu = 0; pu < NPU; pu++) {
				const int pair = tid / tpp + pu * PCG5_BLOCK;
				if (!(pair < npairs && (tid % tpp) == 0 && (pu == 0 || tpp == 1))) continue;
				const int li = pair / 6, comp = pair - 6 * li;
				const int dl = s_diag[li];
				const T ri = s_r[6 * (size_t)dl + comp];
				const T ui = s_v[6 * (size_t)dl + comp];
				const T wv1 = wacc[pu] + ui;                                   // A^_ii = I
				const size_t slot = wHalf + (size_t)opar * wStride + 6 * (size_t)(row0 + li) + comp;
				ll_store(a.wBoard + 2 * slot, (double)wv1, otag);
				if (world > 1) {
					unsigned int peers = a.rowPeers[row0 + li];
					while (peers) {
						const int pr = __ffs(peers) - 1;
						peers &= peers - 1;
						ll_store(a.peerW[pr] + 2 * slot, (double)wv1, otag);
					}
				}
				s_q[pair] = (double)ri * (double)ui;
				s_q[nact + pair] = (double)wv1 * (double)ui;
				s_q[2 * nact + pair] = (double)ri * (double)ri;
				if (coarse) {
					const T* Zh = a.dims.zhInSmem ? s_zh + 36 * (size_t)dl + comp : a.Zhat + 36 * (size_t)(row0 + li) + comp;
#pragma unroll
					for (int q = 0; q < 6; q++) s_q[(3 + q) * nact + pair] = (double)(Zh[6 * q] * wv1);   // (Z^^T w)(q) = sum_comp Z^(comp,q) w(comp)
				}
			}
			__syncthreads();
			PCG_T(t7);
			for (int word = wid; word < NP; word += PCG5_BLOCK / 32) {
				double v = 0;
				for (int i = lane; i < nact; i += 32) v += s_q[word * nact + i];
				v = warp_sum(v);
				if (lane < PCG5_REPL) ll_store(a.pBoard + 2 * (pHalf + (size_t)opar * pStride + ((size_t)lane * G + lc) * NP + word), v, otag);
			}
			PCG_T(t8);
			PCG_ACC(3, t4, t5); PCG_ACC(4, t5, t6); PCG_ACC(5, t6, t7); PCG_ACC(6, t7, t8);
			// s_q / s_cc are rewritten only after the next pass's __syncthreads
		}
	}
	// a rank that gave up tells the others, so that nobody waits for its words
	if (status == 3 && world > 1 && tid < world) atomicExch(&a.peerCtl[tid]->abort, 1);
	// ---- x = L^-T y for the own rows ----
	__syncthreads();
	for (int wi = tid; wi < nrows * 6; wi += PCG5_BLOCK) {
		const int li = wi / 6, r = wi % 6;
		const T* Li = a.Linv + 36 * (size_t)(row0 + li);
		T s = T(0);
		for (int c = r; c < 6; c++) s += Li[r * 6 + c] * s_y[6 * li + c];   // (L^-T)(r,c) = Li(c,r)
		a.x[6 * (size_t)(row0 + li) + r] = s;
	}
#ifdef CUBA_PCG_TIMING
	if (tid == 0 && a.timing) { for (int i = 0; i < 7; i++) a.timing[(size_t)lc * 8 + i] = tacc[i]; a.timing[(size_t)lc * 8 + 7] = it; }
#endif
	if (lc == 0 && tid == 0) {
		a.status->iters = it; a.status->status = status; a.status->rz0 = rho0; a.status->rz = rho;
		// every rank leaves at the same pass (identical scalars) -> identical tag bases for the next solve (k_pcg5_commit)
		a.ctl->advance = (unsigned int)(kExit + 3);
	}
}

template <typename T, bool BIG = false>
__global__ void __launch_bounds__(PCG5_BLOCK, 1) k_pcg5(const Pcg5Args<T> a) { pcg5_body<T, BIG>(a, blockIdx.x); }

// W ranks emulated on one GPU (cuba_debug_pcg5_ranks): one cooperative launch of W * G CTAs, CTA b acting as CTA b % G of rank
// b / G with that rank's arguments args[b / G].  The ranks exchange through device memory only, as on W GPUs.
template <typename T, bool BIG>
__global__ void __launch_bounds__(PCG5_BLOCK, 1) k_pcg5_ranks(const Pcg5Args<T>* args, int G) { pcg5_body<T, BIG>(args[blockIdx.x / G], blockIdx.x % G); }

// between solves: move the tag base past every tag the finished solve used, flip the solve parity, clear the breakdown counter
__global__ void k_pcg5_commit(Pcg5Ctl* ctl)
{
	ctl->tagBase += ctl->advance;
	ctl->solve += 1;
	ctl->nbad = 0;
	ctl->advance = 0;
}

}  // namespace cuba_b200
