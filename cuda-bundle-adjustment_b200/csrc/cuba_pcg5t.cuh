// cuba_pcg5t.cuh -- k_pcg5 (cuba_pcg5.cuh: same mathematics, same LL-word exchange, same boards and tags) in the launch shape
// tuned for ONE GPU whose reduced system fits registers + shared memory (ba_kitti_00 class: <= 512 + cached blocks per CTA):
//   * 512 threads with one register-resident block each (cuba_pcg5.cuh: 256 threads, two blocks): twice the warps to hide the
//     shared-memory and L2 latencies of the short phases between the exchanges;
//   * the coarse residual is advanced first and this CTA's rows of c = Ac^-1 rc are published BEFORE r, s, p, y are advanced, so the
//     words cross the L2 while the CTA still has work to do;
//   * the three scalars are summed by three warps (one each) instead of by all sixteen; the 3 + 6K partial products of the
//     (row, component) threads are added by warp butterflies instead of through a shared-memory staging array;
//   * K = 1, 2 or 3 aggregates per CTA on the coarse level (k_pcg5: one per group of gs CTAs);
//   * one block per thread and product round (the register blocks, then the cached ones), the row sums accumulating over the
//     rounds: 512 staging slots instead of 1 024;
//   * Z^ of the needed columns in shared memory in fp32, the polled partial words behind the polled w inside the product staging,
//     and the needed column (not its six board offsets) per w entry: what makes room for the K = 2 slice of Ac^-1.  The rounded
//     Z^ is the prolongator in both places of the iteration and in rc0 (k_pcg5_prep_rows rounds the global copy), so
//     M^-1 = I + Z^ Ac^-1 Z^^T stays symmetric positive definite and rc stays Z^^T r;
// cuba_pcg5.cuh keeps the multi-GPU and large-graph shape: the same source restructured to serve both shapes ran slower on the
// streamed (BIG) path, so the shapes live in two files.
// The engine picks this kernel for world == 1 solves whose blocks fit on chip (CUBA_PCG5_LEGACY=1 forces the other one).
#pragma once

#include "cuba_pcg5.cuh"

namespace cuba_b200 {
namespace p5t {

// the launch shape
struct Pcg5Shape {
	static constexpr int BLOCK = 512;
	static constexpr int BPT = 1;                      // register-resident A^ blocks per thread
	static constexpr int REGBLK = BLOCK * BPT;         // 512, as in cuba_pcg5.cuh (PCG5_REGBLK)
	static constexpr int CPT = 1;                      // blocks per thread and product round
	static constexpr int CHUNK = BLOCK * CPT;
	static constexpr int PCH = 3;                      // polled words in flight per thread
};

// aggregates per CTA the engine tries first (then fewer, until the plan exists and the shared memory fits).  1: on ba_kitti_00
// (one H100 80GB HBM3, 700 W limit) K = 2 fits with every Z^ and all but 22 of the 182 cached blocks of the fullest CTA on chip and
// cuts the iterations per LM step from 1560 to 1251, but an iteration takes 14.5 instead of 9.8 us (every phase grows: 15
// instead of 9 partial words, 12 instead of 6 rows of Ac^-1 over 1584 instead of 792 columns; DESIGN.md section 7) and a coarse
// rebuild 1.6 instead of 0.5 ms: 24.4 instead of 21.6 ms per step.  K = 2 pays below about 11.4 us per iteration.
constexpr int DEFAULT_APC = 1;

struct Pcg5Dims {
	int capBlocks, needMax, maxRows, nc, maxNeedAgg, zhInSmem;
	int sliceRows; // rows of the inverse coarse matrix this CTA multiplies: ceil(nc / G)
	int npv;      // max(G * NP, world * NR): polled partial / summary words
	int nls;      // NR: words of a rank summary
	int ccCap;    // slots per component of the block-product staging: the shape's CHUNK, or less when a CTA never owns that many blocks
	int sqWords;  // doubles of the partial-product staging: 9 * maxRows * 6
};

// Pcg5Dims::ccCap of a plan: the shape's CHUNK, or less when a CTA never owns that many blocks (Pcg5Layout sizes the storage for
// the polled words it also holds)
inline int pcg5t_cc_cap(int blkMax)
{
	return blkMax >= Pcg5Shape::CHUNK ? Pcg5Shape::CHUNK : std::max((blkMax + 31) / 32 * 32, 32);
}

// shared-memory carve-up, one definition for the host (size) and the device (pointers)
template <typename T>
struct Pcg5Layout {
	size_t blk, r, s, u, p, y, cc, rc, c, zh, pv, ls, sq, ai, loc, rowPtr, col, own, nagg, alist, diag, total;
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
		// block-product staging; between the passes the polled w entries of the needed columns and, behind them, the polled
		// partial words (both double): they are consumed before the next products are staged
		const size_t polled = (size_t)d.needMax * 6 + (size_t)d.npv, staged = (size_t)d.ccCap * 6;
		cc = take((polled > staged ? polled : staged) * sizeof(double), 8);
		pv = cc + (size_t)d.needMax * 6 * sizeof(double);
		rc = take((size_t)d.nc * sizeof(T), 8);
		c = take((size_t)d.maxNeedAgg * 6 * sizeof(T), 8);
		zh = take(d.zhInSmem ? (size_t)d.needMax * 36 * sizeof(float) : 0, 8);
		ls = take((size_t)d.nls * sizeof(double), 8);
		sq = take((size_t)d.sqWords * sizeof(double), 8);           // nine products of every (row, component) thread
		ai = take((size_t)d.sliceRows * d.nc * sizeof(float), 16);
		loc = take((size_t)d.capBlocks * sizeof(int), 4);
		rowPtr = take(((size_t)d.maxRows + 1) * sizeof(int), 4);
		col = take((size_t)d.needMax * sizeof(int), 4);
		own = take((size_t)d.needMax * sizeof(int), 4);
		nagg = take((size_t)d.needMax * sizeof(int), 4);
		alist = take((size_t)d.maxNeedAgg * sizeof(int), 4);
		diag = take((size_t)d.maxRows * sizeof(int), 4);
		total = (o + 15) / 16 * 16;
	}
};

// entries of the coarse search direction sc = wc + beta sc a thread keeps in registers (entry tid + i BLOCK in slot i; only the thread
// that advances rc(q) ever reads sc(q)): a plan needs nc <= BLOCK * pcg5t_nsc(K)
__host__ __device__ constexpr int pcg5t_nsc(int K) { return 2 * K; }

// blocks of a CTA that a plan with K > 1 aggregates per CTA may leave to the global copy (read from L2 in every pass) to make room
// for the K-fold slice of Ac^-1: one warp's share of a product round
constexpr int MAX_STREAMED_BLOCKS = 32;

// Sizes the caches of a plan (every other field of `t` set) for `budget` bytes of shared memory: capBlocks and zhInSmem.
// One aggregate per CTA: every block past the registers is cached (a solve that streams blocks is cuba_pcg5.cuh's BIG shape), Z^
// if it still fits.  Several: Z^ is cached and at most MAX_STREAMED_BLOCKS blocks are not.  False: the plan does not fit.
template <typename T>
inline bool pcg5t_fit(Pcg5Dims& t, int blkMax, int aggsPerCta, size_t budget)
{
	const size_t per = 36 * sizeof(T) + sizeof(int);              // s_blk + s_loc
	const size_t want = blkMax > Pcg5Shape::REGBLK ? (size_t)(blkMax - Pcg5Shape::REGBLK) : 0;
	t.capBlocks = 0; t.zhInSmem = 0;
	if (t.nc > Pcg5Shape::BLOCK * pcg5t_nsc(aggsPerCta)) return false;
	const size_t base = Pcg5Layout<T>(t).total + 64;              // + what the alignment of the regions behind s_blk can add
	const size_t zh = (size_t)t.needMax * 36 * sizeof(float);
	if (aggsPerCta > 1) {
		if (base + zh > budget) return false;
		const size_t cap = std::min(want, (budget - base - zh) / per);
		if (want - cap > (size_t)MAX_STREAMED_BLOCKS) return false;
		t.capBlocks = (int)cap; t.zhInSmem = 1;
		return true;
	}
	if (base + want * per > budget) return false;
	t.capBlocks = (int)want;
	t.zhInSmem = base + want * per + zh <= budget ? 1 : 0;
	return true;
}

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
	const int* aggRow;      // [A+1] first row of every aggregate (read for the K > 1 aggregates of a CTA)
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


// Polls `n` LL words (slot of item i given by slotOf(i)) and hands every value to put(i, v); PCG5_PCH loads of a thread are in
// flight together.  Returns false when the solve was aborted (a peer vanished: spin limit).
template <int KB, int PCG5_PCH, typename SlotOf, typename Put>
__device__ __forceinline__ bool ll_poll_each(int n, SlotOf slotOf, Put put, unsigned int tag, Pcg5Ctl* ctl)
{
	constexpr int PCG5_BLOCK = KB;                      // (shadows the legacy constant inside this function)
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
				if (ll_decode(lo[u], hi[u], tag, v)) { put(base + u * PCG5_BLOCK + tid, v); pend &= ~(1u << u); }
			}
			if ((spin & 1023u) == 1023u) {
				if (*(volatile int*)&ctl->abort) return false;
				if (spin >= PCG3_SPIN_LIMIT) { atomicExch(&ctl->abort, 1); return false; }
			}
		}
	}
	return true;
}
template <int KB, int KPCH, typename SlotOf>
__device__ __forceinline__ bool ll_poll_many(int n, SlotOf slotOf, double* dst, unsigned int tag, Pcg5Ctl* ctl)
{
	return ll_poll_each<KB, KPCH>(n, slotOf, [dst](int i, double v) { dst[i] = v; }, tag, ctl);
}

// partial words of a CTA: gamma, delta, rho, then Z^^T w of each of its K aggregates
__host__ __device__ constexpr int pcg5t_np(int K) { return 3 + 6 * K; }

// K aggregates per CTA on the coarse level (one GPU; K > 1 needs gs == 1): aggregate K cta + j = the j-th of K contiguous groups
// of the CTA's rows.  The coarse space grows K-fold (fewer iterations), a CTA publishes 3 + 6K partial words and multiplies 6K rows
// of Ac^-1.
template <typename T, int K>
__global__ void __launch_bounds__(Pcg5Shape::BLOCK, 1) k_pcg5t(const Pcg5Args<T> a)
{
	using Shape = Pcg5Shape;
	// the names of cuba_pcg5.cuh's constants, bound to this shape
	constexpr int PCG5_BLOCK = Shape::BLOCK, PCG5_BPT = Shape::BPT, PCG5_CPT = Shape::CPT, PCG5_CHUNK = Shape::CHUNK, PCG5_PCH = Shape::PCH;
	constexpr int NPK = pcg5t_np(K);
	constexpr int NSC = pcg5t_nsc(K);
	constexpr int PPCH = K == 1 ? PCG5_PCH : 2 * K;        // polled partial words in flight per thread: G (3 + 6K) in one round on 132 CTAs
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const Pcg5Layout<T> lay(a.dims);
	const int capBlocks = a.dims.capBlocks, nc = a.dims.nc, ccCap = a.dims.ccCap;
	T* s_blk = reinterpret_cast<T*>(smem_raw + lay.blk);            // [36][capBlocks] blocks past the registers, element-major
	T* s_r = reinterpret_cast<T*>(smem_raw + lay.r);                // [needMax][6] residual of the needed columns
	T* s_s = reinterpret_cast<T*>(smem_raw + lay.s);                // [needMax][6] s = w + beta s
	T* s_u = reinterpret_cast<T*>(smem_raw + lay.u);                // [needMax][6] u = M^-1 r
	T* s_p = reinterpret_cast<T*>(smem_raw + lay.p);                // [maxRows][6]
	T* s_y = reinterpret_cast<T*>(smem_raw + lay.y);                // [maxRows][6]
	T* s_cc = reinterpret_cast<T*>(smem_raw + lay.cc);              // [6][ccCap] block products, component-major
	double* s_w = reinterpret_cast<double*>(smem_raw + lay.cc);     // polled w entries of the needed columns (same storage, other phase)
	T* s_rc = reinterpret_cast<T*>(smem_raw + lay.rc);              // [nc] coarse residual Z^^T r
	T* s_c = reinterpret_cast<T*>(smem_raw + lay.c);                // [maxNeedAgg][6]
	float* s_zh = reinterpret_cast<float*>(smem_raw + lay.zh);      // [needMax][36] Z^ of the needed columns
	double* s_pv = reinterpret_cast<double*>(smem_raw + lay.pv);    // polled partials, later polled rank summaries (behind s_w)
	double* s_ls = reinterpret_cast<double*>(smem_raw + lay.ls);    // [NR] this rank's summary
	float* s_ai = reinterpret_cast<float*>(smem_raw + lay.ai);      // [nagg*6][nc] slices of AcInv
	int* s_loc = reinterpret_cast<int*>(smem_raw + lay.loc);
	int* s_rowPtr = reinterpret_cast<int*>(smem_raw + lay.rowPtr);
	int* s_col = reinterpret_cast<int*>(smem_raw + lay.col);        // [needMax] the needed columns: w entry (c, comp) is word 6 s_col[c] + comp of a board
	int* s_own = reinterpret_cast<int*>(smem_raw + lay.own);
	int* s_nagg = reinterpret_cast<int*>(smem_raw + lay.nagg);
	int* s_alist = reinterpret_cast<int*>(smem_raw + lay.alist);
	int* s_diag = reinterpret_cast<int*>(smem_raw + lay.diag);
	__shared__ int s_abort;

	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	const int G = a.G, lc = blockIdx.x, cta = a.rank * G + lc, world = a.world;
	const bool coarse = a.A > 0;
	const int Aloc = coarse ? G / a.gs : 0;             // aggregates hosted by one rank (gs divides G)
	const int NP = coarse ? NPK : 3, NR = 3 + 6 * Aloc;
	const int row0 = a.ctaRow[cta], row1 = a.ctaRow[cta + 1], nrows = row1 - row0;
	// first local row of this CTA's aggregates 1 .. K-1
	int aggCut[K > 1 ? K - 1 : 1];
#pragma unroll
	for (int j = 0; j + 1 < K; j++) aggCut[j] = coarse ? a.aggRow[cta * K + j + 1] - row0 : nrows;
	const int need0 = a.needPtr[cta], nneed = a.needPtr[cta + 1] - need0;
	const int blk0 = a.fRowPtr[row0], nblkCta = a.fRowPtr[row1] - blk0;
	constexpr int REGBLK = Shape::REGBLK;
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
		s_col[i] = j;
		s_own[i] = (j >= row0 && j < row1) ? j - row0 : -1;
		if (coarse) s_nagg[i] = a.needAgg[need0 + i];
	}
	if (coarse) {
		const int na0 = a.naPtr[cta];
		nagg = a.naPtr[cta + 1] - na0;
		for (int i = tid; i < nagg; i += PCG5_BLOCK) s_alist[i] = a.naList[na0 + i];
		for (int i = tid; i < nc; i += PCG5_BLOCK) s_rc[i] = a.rc0[i];
	}
	for (int i = tid; i < nrows * 6; i += PCG5_BLOCK) { s_p[i] = T(0); s_y[i] = T(0); }
	__syncthreads();
	for (int i = tid; i < nneed; i += PCG5_BLOCK) if (s_own[i] >= 0) s_diag[s_own[i]] = i;
	if (coarse) {
		if (a.dims.zhInSmem)
			for (int wi = tid; wi < nneed * 36; wi += PCG5_BLOCK) s_zh[wi] = (float)__ldcg(a.Zhat + 36 * (size_t)a.needCol[need0 + wi / 36] + (wi % 36));
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
			if (n < nblkCta) {
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
				// past the shared-memory cache (the engine sizes this shape so that it does not happen): the global copy, element-major
				// inside this CTA's slice
				for (int e = 0; e < 36; e++) a.fHat[overBase + (size_t)e * nover + (m - ncached)] = out[e];
			}
		}
	}
	for (int wi = tid; wi < nneed * 6; wi += PCG5_BLOCK) {
		s_r[wi] = a.R0[6 * (size_t)s_col[wi / 6] + (wi % 6)];
		s_s[wi] = T(0);
		s_u[wi] = T(0);
	}
	__syncthreads();

	T scReg[NSC];
#pragma unroll
	for (int i = 0; i < NSC; i++) scReg[i] = T(0);
	int status = 1, it = 0, kExit = 0;
	double gamma = 0, rho0 = 0, rho = 0, alpha = 0, beta = 0;
#ifdef CUBA_PCG_TIMING
	long long tacc[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
#endif
	int tpp = 1;                                         // threads per (row, component) pair of the row sums, a power of two
	while (tpp < 8 && nrows * 6 * tpp * 2 <= PCG5_BLOCK) tpp *= 2;
	// s, r of the needed columns, p, y of the own rows (u_k is still in s_u); alpha, beta of the current pass
	auto advance_vectors = [&]() {
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
	};
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
					// two lists, one after the other (one mixed list, the loads of both boards in flight together, was slower on
					// ba_kitti_00 with 256 and with 512 threads)
					bool ok = ll_poll_many<PCG5_BLOCK, PCG5_PCH>(nW, [&](int i) { return wB + 2 * (size_t)(6 * s_col[i / 6] + (i % 6)); }, s_w, tag, a.ctl);
					ok = ok && ll_poll_many<PCG5_BLOCK, PPCH>(nPl, [&](int i) { return pB + 2 * (size_t)i; }, s_pv, tag, a.ctl);
					if (!ok) s_abort = 1;
				}
				__syncthreads();
				PCG_T(t1);
				if (s_abort) { status = 3; break; }
				double gnew, delta, rnew;
				if (world == 1) {
					// ---- one GPU, 16 warps: three of them add one scalar each over the CTAs (every warp adding all three, as k_pcg5 does,
					//      keeps the shared-memory and shuffle pipes busy for ~2 000 cycles); the others meet them at the barrier ----
					if (wid < 3) {
						double v = 0;
						for (int c = lane; c < G; c += 32) v += s_pv[c * NP + wid];
						v = warp_sum(v);
						if (lane == 0) s_ls[wid] = v;
					}
					__syncthreads();
					gnew = s_ls[0]; delta = s_ls[1]; rnew = s_ls[2];
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
					const bool ok = ll_poll_many<PCG5_BLOCK, PCG5_PCH>(world * NR, [&](int i) { return rB + 2 * (size_t)i; }, s_pv, tag, a.ctl);
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
				// ---- advance s, r (needed columns), p, y (own rows; u_k is still in s_u) and the coarse residual: the coarse
				//      residual first -- its product with Ac^-1 is published before r, s, p, y are advanced, so that the words
				//      cross the L2 while this CTA still has work to do ----
				if (!coarse) advance_vectors();
				if (coarse)
#pragma unroll
					for (int i = 0; i < NSC; i++) {
						const int q = tid + i * PCG5_BLOCK;
						if (q >= nc) break;
						// global aggregate q/6 = rank r, local aggregate al
						double wcv;
						if (world > 1) wcv = s_pv[(q / (6 * Aloc)) * NR + 3 + (q % (6 * Aloc))];
						else {
							// aggregate ag: part j of the gs CTAs from c0 on (K == 1: j = 0; K > 1: gs = 1)
							const int ag = q / 6, comp = q - 6 * ag, c0 = ag / K * a.gs, j = ag - ag / K * K;
							wcv = 0;
							for (int c = c0; c < c0 + a.gs; c++) wcv += s_pv[c * NP + 3 + 6 * j + comp];
						}
						const T sc = (T)wcv + (T)beta * scReg[i];
						scReg[i] = sc;
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
				if (k >= 0) advance_vectors();
				{
					const unsigned long long* cR = cB + 2 * ((size_t)rep * nc);
					double* cdst = sizeof(T) == 8 ? reinterpret_cast<double*>(s_c) : s_pv;
					const bool ok = ll_poll_many<PCG5_BLOCK, PCG5_PCH>(nagg * 6, [&](int i) { return cR + 2 * (size_t)(s_alist[i / 6] * 6 + (i % 6)); }, cdst, ctag, a.ctl);
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
						const float* Zh = s_zh + 36 * (size_t)c + comp;
#pragma unroll
						for (int q = 0; q < 6; q++) u += (T)Zh[6 * q] * cc[q];
					} else {
						const T* Zh = a.Zhat + 36 * (size_t)s_col[c] + comp;
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
			constexpr int NPU = 1;                                // (row, component) pairs per thread: nrows * 6 <= BLOCK
			T wacc[NPU];
#pragma unroll
			for (int pu = 0; pu < NPU; pu++) wacc[pu] = T(0);
			const int npairs = nrows * 6;
			for (int cs = 0; cs < nblkCta; cs += PCG5_CHUNK) {
				if (cs > 0) __syncthreads();
#pragma unroll
				for (int u = 0; u < PCG5_CPT; u++) {
					const int n = cs + u * PCG5_BLOCK + tid;
					T y[6] = { T(0), T(0), T(0), T(0), T(0), T(0) };
					if (u < PCG5_BPT && cs == 0) {
						const int ur = u < PCG5_BPT ? u : 0;
						if (myLoc[ur] >= 0) {
							const T* rj = s_v + 6 * (size_t)myLoc[ur];
#pragma unroll
							for (int c = 0; c < 6; c++) {
								const T rc = rj[c];
#pragma unroll
								for (int r = 0; r < 6; r++) y[r] += breg[ur][c * 6 + r] * rc;
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
							} else {
								// the few blocks a K > 1 plan leaves to the global copy: written by this CTA before the first pass and never
								// again, so they may stay in the L1 (plain loads)
								const T* B = a.fHat + overBase + (m - ncached);
#pragma unroll 1
								for (int c = 0; c < 6; c++) {
									const T rc = rj[c];
#pragma unroll
									for (int r = 0; r < 6; r++) { y[r] += *B * rc; B += nover; }
								}
							}
						}
					}
					if (u * PCG5_BLOCK + tid < ccCap) {
#pragma unroll
						for (int r = 0; r < 6; r++) s_cc[r * ccCap + u * PCG5_BLOCK + tid] = y[r];
					}
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
						const T* col = s_cc + comp * ccCap;
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
#ifdef CUBA_PCG_TIMING
			long long t7 = 0;
#endif
			// Every (row, component) thread keeps its NPK products in registers; a butterfly adds them over the warp, lane 0 leaves the
			// warp's sums in shared memory and NP x REPL threads add the warps in a fixed order and publish the replicas.
			double* s_q = reinterpret_cast<double*>(smem_raw + lay.sq);   // [warps][NPK]; rewritten only after the next pass's barriers
			double q9[NPK];
#pragma unroll
			for (int w = 0; w < NPK; w++) q9[w] = 0.0;
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
				q9[0] += (double)ri * (double)ui;
				q9[1] += (double)wv1 * (double)ui;
				q9[2] += (double)ri * (double)ri;
				if (coarse) {
					const float* ZhS = s_zh + 36 * (size_t)dl + comp;
					const T* ZhG = a.Zhat + 36 * (size_t)(row0 + li) + comp;
					int ja = 0;                                                    // the row's aggregate within this CTA
#pragma unroll
					for (int j = 0; j + 1 < K; j++) ja += li >= aggCut[j] ? 1 : 0;
#pragma unroll
					for (int q = 0; q < 6; q++) {
						const double z = (double)((a.dims.zhInSmem ? (T)ZhS[6 * q] : ZhG[6 * q]) * wv1);   // (Z^^T w)(q) = sum_comp Z^(comp,q) w(comp)
#pragma unroll
						for (int j = 0; j < K; j++) if (ja == j) q9[3 + 6 * j + q] += z;
					}
				}
			}
			// only the lanes tid % tpp == 0 hold products: the butterfly starts at distance tpp (the shorter ones would add zeros)
#pragma unroll
			for (int w = 0; w < NPK; w++) if (w < NP) {
#pragma unroll
				for (int o = 16; o > 0; o >>= 1) if (o >= tpp) q9[w] += __shfl_xor_sync(0xffffffffu, q9[w], o);
			}
			if (lane == 0) {
#pragma unroll
				for (int w = 0; w < NPK; w++) if (w < NP) s_q[wid * NPK + w] = q9[w];
			}
			__syncthreads();
#ifdef CUBA_PCG_TIMING
			t7 = clock64();
#endif
			if (tid < NP * PCG5_REPL) {
				const int word = tid / PCG5_REPL, rp = tid - word * PCG5_REPL;
				double v = 0;
#pragma unroll
				for (int w8 = 0; w8 < PCG5_BLOCK / 32; w8++) v += s_q[w8 * NPK + word];
				ll_store(a.pBoard + 2 * (pHalf + (size_t)opar * pStride + ((size_t)rp * G + lc) * NP + word), v, otag);
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


}  // namespace p5t
}  // namespace cuba_b200
