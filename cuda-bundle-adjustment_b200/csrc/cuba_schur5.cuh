// cuba_schur5.cuh -- landmark-tile Schur complement on the fp64 tensor pipe (DMMA m8n8k4).
//
// What bounds k_schur3: every one of the 2.3 M block products of a ba_kitti_00-sized
// graph gathers two 144-byte Hpl blocks and a 72-byte inverse from L2 -- 0.8 GB per launch, 7x the algorithmic bytes, through
// L1TEX -- because the products are walked destination by destination while Hpl is stored landmark by landmark.
// Here the walk follows the storage: a CTA owns a tile of consecutive landmarks (its own tiling: windows of 448 edges, <= 512 Hpl
// blocks, brings the tile's contiguous Hpl range into shared memory ONCE (coalesced), inverts the tile's Hll blocks, factors the
// inverse  inv(Hll + lambda I) = L L^T  (3x3 Cholesky) and turns every staged block into V_i = Hpl_i L in place, so that
// Hpl_i inv Hpl_j^T = V_i V_j^T needs ONE staged array.  Then one WARP per (tile, destination block) segment accumulates the
// segment's products  C += V_i V_j^T  with one `mma.sync.m8n8k4.f64` each: A fragment = V_i (6x3 padded to 8x4), B fragment
// = V_j^T (3x6 padded to 4x8; column 6 carries u = L^T bl of the landmark on diagonal destinations, so the bsc contribution
// Hpl_i inv bl = V_i u rides in the same instruction), both read from shared memory with ONE 8-byte load per lane.
// The 6x6 (+6) partial of the segment goes to a buffer; k_schur_reduce adds the partials of every destination in a
// fixed order (tiles ascending) and applies the Hpp / lambda / sign epilogue.  No atomics, bit-reproducible.
// Replaces computeBschureKernel / initializeHschurKernel / computeHschureKernel (reference src/cuda_block_solver.cu:933-977).
#pragma once

#include "cuba_kernels.cuh"

namespace cuba_b200 {

// landmark tiles of the Schur stage: landmarks [l0, l1), edges [e0, e1), poses [pose0, pose0 + poseN), Hpl blocks [h0, h1)
struct TileInfo { int l0, l1, e0, e1, pose0, poseN, h0, h1; };   // h0/h1: Hpl block index at e0 / e1

__global__ void k_tile_info3(const int* __restrict__ tilePtr, const int* __restrict__ tileLm, const int* __restrict__ ip,
	const int* __restrict__ hpl, int eLocal, int nhplLocal, int ntiles, TileInfo* info)
{
	__shared__ int s_min, s_max;
	if (threadIdx.x == 0) { s_min = 0x7fffffff; s_max = -1; }
	__syncthreads();
	const int l0 = tileLm[blockIdx.x], l1 = tileLm[blockIdx.x + 1];
	const int e0 = tilePtr[l0], e1 = tilePtr[l1];
	int mn = 0x7fffffff, mx = -1;
	for (int e = e0 + threadIdx.x; e < e1; e += blockDim.x) { const int p = ip[e] & 0x7fffffff; mn = p < mn ? p : mn; mx = p > mx ? p : mx; }
	atomicMin(&s_min, mn); atomicMax(&s_max, mx);
	__syncthreads();
	if (threadIdx.x == 0) {
		auto rankAt = [&](int e) { if (e >= eLocal) return nhplLocal; const int x = hpl[e]; return x >= 0 ? x : -1 - x; };
		TileInfo ti;
		ti.l0 = l0; ti.l1 = l1; ti.e0 = e0; ti.e1 = e1;
		ti.pose0 = s_max >= 0 ? s_min : 0; ti.poseN = s_max >= 0 ? s_max - s_min + 1 : 0;
		ti.h0 = rankAt(e0); ti.h1 = rankAt(e1);
		info[blockIdx.x] = ti;
	}
}

namespace schur5 {

constexpr int TL = 512;            // Hpl blocks staged per tile
constexpr int BS = 21;             // doubles per staged block: V (6x3, column-major) followed by u (3)
constexpr int WINDOW = 448;        // edges per tile window of the structure builder: leaves 64 slots for the last landmark's tail
constexpr int WARPS = 8;
constexpr int PW = 42;             // doubles per partial: 36 (block) + 6 (bsc part, zero off the diagonal)

// ---- (tile, destination) segments of the block products, built once per structure (Engine::setup_schur5) ----

// key = (tile << 32) | destination block, for every real product of the destination-sorted list
__global__ void k_keys(const int* __restrict__ prodPtr, int nblk, const int* __restrict__ prodI, int N, const TileInfo* __restrict__ info, int ntiles,
	unsigned long long* key, int* val)
{
	const int n = blockIdx.x * blockDim.x + threadIdx.x;
	if (n >= N) return;
	val[n] = n;
	const int i = prodI[n];
	if (i < 0) { key[n] = ~0ull; return; }
	int lo = 0, hi = ntiles - 1;                 // first tile with h1 > i
	while (lo < hi) { const int mid = (lo + hi) >> 1; if (info[mid].h1 > i) hi = mid; else lo = mid + 1; }
	const int tile = lo;
	lo = 0; hi = nblk - 1;                       // destination k: last k with prodPtr[k] <= n
	while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (prodPtr[mid] <= n) lo = mid; else hi = mid - 1; }
	key[n] = ((unsigned long long)(unsigned)tile << 32) | (unsigned)lo;
}

__global__ void k_heads(const unsigned long long* __restrict__ key, int N, int* head)
{
	const int n = blockIdx.x * blockDim.x + threadIdx.x;
	if (n >= N) return;
	head[n] = (key[n] != ~0ull && (n == 0 || key[n] != key[n - 1])) ? 1 : 0;
}

struct Counts { int nseg; int nvalid; };

__global__ void k_counts(const unsigned long long* __restrict__ key, const int* __restrict__ head, const int* __restrict__ segId, int N, Counts* out)
{
	if (blockIdx.x != 0 || threadIdx.x != 0) return;
	out->nseg = N > 0 ? segId[N - 1] + head[N - 1] : 0;
	int lo = 0, hi = N;                          // first sentinel
	while (lo < hi) { const int mid = (lo + hi) >> 1; if (key[mid] == ~0ull) hi = mid; else lo = mid + 1; }
	out->nvalid = lo;
}

__global__ void k_segments(const unsigned long long* __restrict__ key, const int* __restrict__ valSorted, const int* __restrict__ head,
	const int* __restrict__ segId, const int* __restrict__ prodI, const int* __restrict__ prodJ, int N, int nseg, int nvalid,
	int* segStart, int* segTile, int* segDest, int* p2i, int* p2j, unsigned long long* key3, int* val3)
{
	const int n = blockIdx.x * blockDim.x + threadIdx.x;
	if (n > N) return;
	if (n == N) { segStart[nseg] = nvalid; return; }
	if (key[n] == ~0ull) return;
	if (head[n]) {
		const int s = segId[n];
		const int tile = (int)(key[n] >> 32), dest = (int)(key[n] & 0xffffffffu);
		segStart[s] = n; segTile[s] = tile; segDest[s] = dest;
		key3[s] = ((unsigned long long)(unsigned)dest << 32) | (unsigned)tile;
		val3[s] = s;
	}
	const int src = valSorted[n];
	p2i[n] = prodI[src]; p2j[n] = prodJ[src];
}

// ptr[i] = first segment (sorted by the given 32-bit field, ascending) with field >= i
__global__ void k_ptr_from_field(const int* __restrict__ field, int n, int m, int* ptr)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > m) return;
	int lo = 0, hi = n;
	while (lo < hi) { const int mid = (lo + hi) >> 1; if (field[mid] < i) lo = mid + 1; else hi = mid; }
	ptr[i] = lo;
}

__global__ void k_rank(const unsigned long long* __restrict__ key3Sorted, const int* __restrict__ val3Sorted, int nseg, int* segRank, int* rankDest)
{
	const int r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= nseg) return;
	segRank[val3Sorted[r]] = r;
	rankDest[r] = (int)(key3Sorted[r] >> 32);
}

struct Smem {
	double V[TL * BS];             // per block: V = Hpl chol(inv(Hll + lambda I)) and u = L^T bl of its landmark:
	                               // C_ij = sum_l V_il V_jl^T needs ONE staged array, the bsc contribution is V_il u_l
	double zero[2];                // what the padding lanes of a fragment read
	double L[TL * 6];              // lower Cholesky factor of the inverse per landmark, 00,10,20,11,21,22
	int lm[TL];                    // local landmark of each block
};

// lower Cholesky factor of a symmetric positive definite 3x3 given as 00,01,02,11,12,22 -> 00,10,20,11,21,22
__device__ __forceinline__ void chol3(const double B[6], double L[6])
{
	L[0] = sqrt(B[0]);
	const double i0 = 1.0 / L[0];
	L[1] = B[1] * i0; L[2] = B[2] * i0;
	L[3] = sqrt(B[3] - L[1] * L[1]);
	L[4] = (B[4] - L[2] * L[1]) / L[3];
	L[5] = sqrt(B[5] - L[2] * L[2] - L[4] * L[4]);
}

// per (tile, destination) segment: first product, product count, rank among the destination-sorted partials,
// flags: bit 0 = diagonal destination, bit 1 = some block of the segment lies past the staged range (slow path)
__global__ void k_seg_records(const int* __restrict__ segStart, const int* __restrict__ segDest, const int* __restrict__ segRank, const int* __restrict__ segTile,
	const int* __restrict__ blkRow, const int* __restrict__ blkCol, const TileInfo* __restrict__ info, const int* __restrict__ p2i, const int* __restrict__ p2j,
	int nseg, int4* rec)
{
	const int s = blockIdx.x * blockDim.x + threadIdx.x;
	if (s >= nseg) return;
	const int k = segDest[s], h0 = info[segTile[s]].h0;
	int flags = blkRow[k] == blkCol[k] ? 1 : 0;
	for (int n = segStart[s]; n < segStart[s + 1]; n++) if (p2i[n] - h0 >= TL || p2j[n] - h0 >= TL) { flags |= 2; break; }
	rec[s] = make_int4(segStart[s], segStart[s + 1] - segStart[s], segRank[s], flags);
}
// operand offsets of every product inside its tile's staged array, in doubles: (block - h0) * BS, both in one word
__global__ void k_prod_offsets(const int* __restrict__ segStart, const int* __restrict__ segTile, const TileInfo* __restrict__ info,
	const int* __restrict__ p2i, const int* __restrict__ p2j, int nseg, int nprod, unsigned int* off)
{
	const int n = blockIdx.x * blockDim.x + threadIdx.x;
	if (n >= nprod) return;
	int lo = 0, hi = nseg - 1;                   // segment of product n: last s with segStart[s] <= n
	while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (segStart[mid] <= n) lo = mid; else hi = mid - 1; }
	const int h0 = info[segTile[lo]].h0;
	const int bi = p2i[n] - h0, bj = p2j[n] - h0;
	const unsigned int oi = bi < TL ? (unsigned)(bi * BS) : 0u, oj = bj < TL ? (unsigned)(bj * BS) : 0u;   // (slow segments do not use them)
	off[n] = oi | (oj << 16);
}

struct Args {
	const double* Hpl; const double* Hll; const double* bl;
	const TileInfo* info; const int* hplLm;
	const int* tileSegPtr; const int4* segRec; const unsigned int* off; const int* p2i; const int* p2j;
	int numL; double lambda;
	double* invHll; double* partial;
};

__global__ void __launch_bounds__(WARPS * 32, 2) k_schur_tiles_mma(const Args a)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, t = blockIdx.x;
	const TileInfo ti = a.info[t];
	const int nb = ti.h1 - ti.h0;
	int nl = ti.l1 - ti.l0;
	if (ti.l0 + nl > a.numL) nl = a.numL - ti.l0;       // the pseudo-landmark of the fixed ones has no Hll
	const int nbs = nb < TL ? nb : TL;
	for (int i = tid; i < nbs * 9; i += WARPS * 32) {
		double x, y;
		ld2(a.Hpl + 18 * (size_t)ti.h0 + 2 * i, x, y);
		const int b = i / 9, e = 2 * (i - 9 * b);
		sm.V[BS * b + e] = x; sm.V[BS * b + e + 1] = y;
	}
	for (int i = tid; i < nbs; i += WARPS * 32) sm.lm[i] = a.hplLm[ti.h0 + i] - ti.l0;
	if (tid < 2) sm.zero[tid] = 0.0;
	for (int j = tid; j < nl; j += WARPS * 32) {
		const double* H = a.Hll + 9 * (size_t)(ti.l0 + j);
		double B[6];
		sym3_inverse<double>(H[0] + a.lambda, H[3], H[6], H[4] + a.lambda, H[7], H[8] + a.lambda, B);
		double* o = a.invHll + 9 * (size_t)(ti.l0 + j);
		o[0] = B[0]; o[1] = B[1]; o[2] = B[2]; o[3] = B[1]; o[4] = B[3]; o[5] = B[4]; o[6] = B[2]; o[7] = B[4]; o[8] = B[5];
		if (j < TL) {
			double L[6];
			chol3(B, L);
#pragma unroll
			for (int k = 0; k < 6; k++) sm.L[6 * j + k] = L[k];
		}
	}
	if (nb <= 0) return;
	__syncthreads();
	// V = Hpl L in place: one (block, row) pair per thread step; (A L)(r,k) = sum_{m>=k} A(r,m) L(m,k); row 0's thread adds u
	for (int w = tid; w < nbs * 6; w += WARPS * 32) {
		const int b = w / 6, r = w - 6 * b;
		const int lml = sm.lm[b];
		double L[6];
		if (lml < TL) {
#pragma unroll
			for (int k = 0; k < 6; k++) L[k] = sm.L[6 * lml + k];
		} else {
			const double* iv = a.invHll + 9 * (size_t)(ti.l0 + lml);
			const double B[6] = { iv[0], iv[3], iv[6], iv[4], iv[7], iv[8] };
			chol3(B, L);
		}
		double* Vb = sm.V + BS * b;
		const double a0 = Vb[r], a1 = Vb[6 + r], a2 = Vb[12 + r];
		Vb[r] = a0 * L[0] + a1 * L[1] + a2 * L[2];
		Vb[6 + r] = a1 * L[3] + a2 * L[4];
		Vb[12 + r] = a2 * L[5];
		if (r == 0) {
			const double* bb = a.bl + 3 * (size_t)(ti.l0 + lml);
			const double b0 = bb[0], b1 = bb[1], b2 = bb[2];
			Vb[18] = L[0] * b0 + L[1] * b1 + L[2] * b2;           // (L^T b)(k) = sum_m L(m,k) b(m)
			Vb[19] = L[3] * b1 + L[4] * b2;
			Vb[20] = L[5] * b2;
		}
	}
	__syncthreads();
	// fragment coordinates of this lane: A[g][q] (q = k), B[q][g] (g = n), C[g][2q], C[g][2q+1]
	const int g = lane >> 2, q = lane & 3;
	const bool inAB = g < 6 && q < 3;
	const int fo = q * 6 + g;                            // offset of element (g, q) in a column-major 6x3 block
	const int s0 = a.tileSegPtr[t], s1 = a.tileSegPtr[t + 1];
	// Software pipeline over this warp's segments (s, s + WARPS, ...): the record of the segment after next and the first 32
	// operand offsets of the next segment are in flight while the current segment is multiplied -- with ~9 products per segment
	// the two dependent L2 round trips (record -> offsets) would otherwise cost more than the products themselves.
	const int4 none = make_int4(0, 0, 0, 0);
	int4 rec = s0 + wid < s1 ? __ldg(a.segRec + s0 + wid) : none;
	int4 recN = s0 + wid + WARPS < s1 ? __ldg(a.segRec + s0 + wid + WARPS) : none;
	unsigned int cur = 0;
	if (s0 + wid < s1 && lane < rec.y) cur = __ldg(a.off + rec.x + lane);
	// operand addresses of this lane: base + (offset of the product's block) * mul -- padding lanes read sm.zero
	const double* aBase = inAB ? sm.V + fo : sm.zero;
	const int aMul = inAB ? 1 : 0;
	for (int s = s0 + wid; s < s1; s += WARPS) {
		const int4 recNN = s + 2 * WARPS < s1 ? __ldg(a.segRec + s + 2 * WARPS) : none;
		unsigned int nxt = 0;
		if (s + WARPS < s1 && lane < recN.y) nxt = __ldg(a.off + recN.x + lane);
		const bool diag = (rec.w & 1) != 0;
		// column 6 of the B fragment carries u on diagonal destinations (there the product pairs a block with itself: the engine
		// runs k_schur3 instead on a graph with a repeated (pose, landmark) pair, whose diagonal destinations also pair two blocks)
		const bool useU = diag && g == 6 && q < 3;
		const double* bBase = inAB ? sm.V + fo : (useU ? sm.V + 18 + q : sm.zero);
		const int bMul = (inAB || useU) ? 1 : 0;
		// four independent accumulator pairs (products u, u+1, u+2, u+3 of every group of four): the chains of dependent
		// shuffle -> shared load -> DMMA overlap; the grouping is fixed, so the sum is reproducible
		double c0 = 0.0, c1 = 0.0, d0 = 0.0, d1 = 0.0, e0 = 0.0, e1 = 0.0, f0 = 0.0, f1 = 0.0;
		const int n0 = rec.x, n1 = rec.x + rec.y;
		if (!(rec.w & 2)) {
			for (int nb0 = n0; nb0 < n1; nb0 += 32) {
				const int nn = n1 - nb0 < 32 ? n1 - nb0 : 32;
				unsigned int my = cur;                            // the first 32 were prefetched
				if (nb0 > n0) { my = 0; if (lane < nn) my = __ldg(a.off + nb0 + lane); }
#define CUBA_S5_STEP(U, C0, C1)                                                                   \
				{                                                                                 \
					const unsigned int o = __shfl_sync(0xffffffffu, my, (U));                     \
					dmma884(C0, C1, aBase[(o & 0xffffu) * aMul], bBase[(o >> 16) * bMul]);        \
				}
				int u = 0;
				for (; u + 4 <= nn; u += 4) {
					CUBA_S5_STEP(u, c0, c1) CUBA_S5_STEP(u + 1, d0, d1) CUBA_S5_STEP(u + 2, e0, e1) CUBA_S5_STEP(u + 3, f0, f1)
				}
				for (; u < nn; u++) CUBA_S5_STEP(u, c0, c1)
#undef CUBA_S5_STEP
			}
			c0 = (c0 + d0) + (e0 + f0); c1 = (c1 + d1) + (e1 + f1);
		} else {
			// a segment with a block past the staged range (a landmark with more observations than the window's slack):
			// every operand straight from global memory, V(g,q) = sum_{m>=q} Hpl(g,m) L(m,q)
			for (int n = n0; n < n1; n++) {
				const int bi = __ldg(a.p2i + n), bj = __ldg(a.p2j + n);
				const int lmg = a.hplLm[bi];
				const double* iv = a.invHll + 9 * (size_t)lmg;
				const double B[6] = { iv[0], iv[3], iv[6], iv[4], iv[7], iv[8] };
				double L[6];
				chol3(B, L);
				const double lq0 = q == 0 ? L[0] : 0.0, lq1 = q == 0 ? L[1] : (q == 1 ? L[3] : 0.0), lq2 = q == 0 ? L[2] : (q == 1 ? L[4] : L[5]);
				double av = 0.0, bv = 0.0;
				if (inAB) {
					const double* gi = a.Hpl + 18 * (size_t)bi;
					const double* gj = a.Hpl + 18 * (size_t)bj;
					av = gi[g] * lq0 + gi[6 + g] * lq1 + gi[12 + g] * lq2;
					bv = gj[g] * lq0 + gj[6 + g] * lq1 + gj[12 + g] * lq2;
				} else if (useU) {
					const double* bb = a.bl + 3 * (size_t)lmg;
					bv = q == 0 ? L[0] * bb[0] + L[1] * bb[1] + L[2] * bb[2] : (q == 1 ? L[3] * bb[1] + L[4] * bb[2] : L[5] * bb[2]);
				}
				dmma884(c0, c1, av, bv);
			}
		}
		// C[g][2q], C[g][2q+1]: the 6x6 block (column-major) and, in column 6, the bsc part
		double* out = a.partial + (size_t)PW * rec.z;
		if (g < 6) {
			if (q < 3) { out[(2 * q) * 6 + g] = c0; out[(2 * q + 1) * 6 + g] = c1; }
			else out[36 + g] = c0;
		}
		rec = recN; recN = recNN; cur = nxt;
	}
}

template <typename T>
struct ReduceArgs {
	const T* partial; const int* destSegPtr;
	const T* Hpp; const T* bp;
	const int* blkRow; const int* blkCol; const int* u2f; const int* u2fT;
	int nblk; T lambda; int addDiag;
	T* fVal; T* bsc;
};

// one warp per destination block: fixed-order sum of its partials (tiles ascending), then the Hpp / lambda / sign epilogue
template <typename T>
__global__ void __launch_bounds__(128) k_schur_reduce(const ReduceArgs<T> a)
{
	const int lane = threadIdx.x & 31;
	const int k = blockIdx.x * 4 + (threadIdx.x >> 5);
	if (k >= a.nblk) return;
	const int ra = a.blkRow[k], cb = a.blkCol[k];
	const bool diag = ra == cb;
	const int r0 = a.destSegPtr[k], r1 = a.destSegPtr[k + 1];
	for (int e = lane; e < PW; e += 32) {
		T s = T(0);
		for (int r = r0; r < r1; r++) s += a.partial[(size_t)PW * r + e];
		if (e < 36) {
			const int c = e / 6, rr = e - 6 * c;
			T val = -s;
			if (diag && a.addDiag) val += a.Hpp[36 * (size_t)ra + e] + (rr == c ? a.lambda : T(0));
			a.fVal[36 * (size_t)a.u2f[k] + e] = val;
			if (!diag) a.fVal[36 * (size_t)a.u2fT[k] + rr * 6 + c] = val;
		} else if (diag) {
			const int rr = e - 36;
			a.bsc[6 * (size_t)ra + rr] = (a.addDiag ? a.bp[6 * (size_t)ra + rr] : T(0)) - s;
		}
	}
}

}  // namespace schur5
}  // namespace cuba_b200
