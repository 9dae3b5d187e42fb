// cuba_structure_gpu.cuh -- device-side construction of every index structure (the GPU twin of
// cuba_structure.cpp; the two must agree bit for bit, tests/test_gpu_parity.py checks it).
//
// Replaces the reference's host code on the "1: Build Structure" path:
//   CudaBlockSolver::initialize edge flattening order  src/cuda_bundle_adjustment.cpp:202-243 (host)
//   gpu::buildHplStructure                              src/cuda_block_solver.cu:1158-1173 (thrust sort)
//   HschurSparseBlockMatrix::constructFromVertices      src/sparse_block_matrix.cpp:55-133 (host, dense PxP map)
//   gpu::findHschureMulBlockIndices                     cu:979-1000,1175-1190
// Sorting and scans use CUB (part of the CUDA toolkit, like the reference's Thrust); everything else is
// the kernels below.
#pragma once

#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <stdint.h>

namespace cuba_b200 {
namespace sgpu {

constexpr int BLK = 256;
inline int grid_for(long long n) { return (int)((n + BLK - 1) / BLK); }

struct Meta {            // small device->host record, one copy per sync point
	int error;           // 0 ok, 1 index out of range, 2 both ends fixed, 3 landmark without edges
	int nhpl;
	int lmBeg, lmEnd, kBeg, kEnd, hplBase, hplEnd;
	long long nmul;      // number of real block products (without the diagonal dummies)
	int nblk;
	int npe;             // pose-major entries
	int bounds[9];       // first landmark of every rank's shard (world <= 8), bounds[world] = Lall
	int repeats;         // 1: some free pose observes some free landmark through more than one edge
};

// (iL, iP) sort keys of the user-order edges; validates the indices.
__global__ void k_make_keys(int E2, const int* __restrict__ idx2, int E3, const int* __restrict__ idx3, int Pall, int numP, int Lall, int numL,
	unsigned long long* key, int* val, Meta* meta)
{
	const int u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= E2 + E3) return;
	const int ip = u < E2 ? idx2[2 * (size_t)u] : idx3[2 * (size_t)(u - E2)];
	const int il = u < E2 ? idx2[2 * (size_t)u + 1] : idx3[2 * (size_t)(u - E2) + 1];
	if (ip < 0 || ip >= Pall || il < 0 || il >= Lall) { atomicMax(&meta->error, 1); key[u] = ~0ull; val[u] = u; return; }
	if (ip >= numP && il >= numL) atomicMax(&meta->error, 2);
	key[u] = ((unsigned long long)(unsigned)il << 32) | (unsigned)ip;
	val[u] = u;
}

// ptr[i] = first position k in the sorted 64-bit keys with (key >> 32) >= i, for i in [0, n]
__global__ void k_ptr_from_high(const unsigned long long* __restrict__ keys, int nkeys, int n, int* ptr)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > n) return;
	int lo = 0, hi = nkeys;
	while (lo < hi) { const int mid = (lo + hi) >> 1; if ((int)(keys[mid] >> 32) < i) lo = mid + 1; else hi = mid; }
	ptr[i] = lo;
}

// ptr[i] = first position with key32 >= i
__global__ void k_ptr_from_u32(const unsigned int* __restrict__ keys, int nkeys, int n, int* ptr)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > n) return;
	int lo = 0, hi = nkeys;
	while (lo < hi) { const int mid = (lo + hi) >> 1; if ((int)keys[mid] < i) lo = mid + 1; else hi = mid; }
	ptr[i] = lo;
}

// every FREE landmark must have an edge; fixed landmarks may have none (all their observers fixed: the
// reference keeps such vertices, src/cuda_bundle_adjustment.cpp:163-178, and drops only the edges, :212,233)
__global__ void k_check_nonempty(const int* __restrict__ lmPtrG, int numL, Meta* meta)
{
	const int l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l < numL && lmPtrG[l + 1] == lmPtrG[l]) atomicMax(&meta->error, 3);
}

// run pointers used by the landmark tiles: the free landmarks one by one, then ALL fixed landmarks of the
// shard as one pseudo-landmark numL (its edges only contribute chi2 there; Hpp comes from the pose pass)
__global__ void k_tile_ptr(const int* __restrict__ lmPtr, int numL, int eLocal, int* tilePtr)
{
	const int l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l > numL + 1) return;
	tilePtr[l] = l <= numL ? lmPtr[l] : eLocal;
}

__global__ void k_flag_freefree(const unsigned long long* __restrict__ keys, int E, int numP, int numL, int* ff)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= E) return;
	const int il = (int)(keys[k] >> 32), ip = (int)(keys[k] & 0xffffffffu);
	ff[k] = (ip < numP && il < numL) ? 1 : 0;
}

// landmark shard of this rank (balanced by edge count, snapped to landmark boundaries) + sizes
__global__ void k_shard_meta(const int* __restrict__ lmPtrG, int Lall, int E, int rank, int world, const int* __restrict__ ff,
	const int* __restrict__ hplG, Meta* meta)
{
	if (blockIdx.x != 0 || threadIdx.x != 0) return;
	auto bound = [&](int r) {
		if (r <= 0) return 0;
		if (r >= world) return Lall;
		const int target = (int)((long long)E * r / world);
		int lo = 0, hi = Lall + 1;
		while (lo < hi) { const int mid = (lo + hi) >> 1; if (lmPtrG[mid] < target) lo = mid + 1; else hi = mid; }
		return lo < Lall ? lo : Lall;
	};
	const int b0 = bound(rank);
	int b1 = bound(rank + 1);
	if (b1 < b0) b1 = b0;
	meta->lmBeg = b0; meta->lmEnd = b1; meta->kBeg = lmPtrG[b0]; meta->kEnd = lmPtrG[b1];
	{
		int prev = 0;
		for (int r = 0; r <= world && r < 9; r++) { int b = bound(r); if (b < prev) b = prev; meta->bounds[r] = b; prev = b; }
	}
	const int nh = E > 0 ? hplG[E - 1] + ff[E - 1] : 0;
	meta->nhpl = nh;
	meta->hplBase = meta->kBeg < E ? hplG[meta->kBeg] : nh;
	meta->hplEnd = meta->kEnd < E ? hplG[meta->kEnd] : nh;
}

// global Hpl structure (CSC rows + landmark of every block, user edge -> block map)
__global__ void k_hpl_global(const unsigned long long* __restrict__ keys, const int* __restrict__ val, const int* __restrict__ ff,
	const int* __restrict__ hplG, int E, int* hplRowInd, int* hplLmG, int* edge2Hpl)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= E) return;
	const int h = ff[k] ? hplG[k] : -1;
	edge2Hpl[val[k]] = h;
	if (h >= 0) { hplRowInd[h] = (int)(keys[k] & 0xffffffffu); hplLmG[h] = (int)(keys[k] >> 32); }
}

__global__ void k_hpl_colptr(const int* __restrict__ lmPtrG, const int* __restrict__ hplG, int E, int numL, int nhpl, int* hplColPtr)
{
	const int l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l > numL) return;
	const int k = lmPtrG[l];
	hplColPtr[l] = k < E ? hplG[k] : nhpl;
}

// landmark-major edge stream of the shard
template <typename T>
__global__ void k_edge_stream(const unsigned long long* __restrict__ keys, const int* __restrict__ val, const int* __restrict__ ff,
	const int* __restrict__ hplG, int kBeg, int eLocal, int hplBase, int E2,
	const double* __restrict__ meas2, const double* __restrict__ om2, const double* __restrict__ meas3, const double* __restrict__ om3,
	int* e_user, int* e_ip, int* e_il, int* e_hpl, T* mx, T* my, T* mz, T* om)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= eLocal) return;
	const int k = kBeg + e, u = val[k];
	const bool stereo = u >= E2;
	e_user[e] = u;
	e_ip[e] = (int)(keys[k] & 0xffffffffu) | (stereo ? (int)0x80000000u : 0);
	e_il[e] = (int)(keys[k] >> 32);
	e_hpl[e] = ff[k] ? hplG[k] - hplBase : -1 - (hplG[k] - hplBase);   // rank among the free-free edges; negative: no block
	if (!stereo) { mx[e] = (T)meas2[2 * (size_t)u]; my[e] = (T)meas2[2 * (size_t)u + 1]; mz[e] = T(0); om[e] = (T)om2[u]; }
	else { const size_t s = (size_t)(u - E2); mx[e] = (T)meas3[3 * s]; my[e] = (T)meas3[3 * s + 1]; mz[e] = (T)meas3[3 * s + 2]; om[e] = (T)om3[s]; }
}

__global__ void k_local_lmptr(const int* __restrict__ lmPtrG, int Lall, int kBeg, int kEnd, int* lmPtr)
{
	const int l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l > Lall) return;
	int v = lmPtrG[l];
	v = v < kBeg ? kBeg : (v > kEnd ? kEnd : v);
	lmPtr[l] = v - kBeg;
}

// tileLm[t] = first landmark (>= lmBeg) whose run starts at or after edge t*tile; tileLm[nt] = lmEnd
__global__ void k_tiles(const int* __restrict__ lmPtr, int lmBeg, int lmEnd, int tile, int nt, int* tileLm)
{
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t > nt) return;
	if (t == nt) { tileLm[t] = lmEnd; return; }
	const int target = t * tile;
	int lo = lmBeg, hi = lmEnd;
	while (lo < hi) { const int mid = (lo + hi) >> 1; if (lmPtr[mid] < target) lo = mid + 1; else hi = mid; }
	tileLm[t] = lo;
}

__global__ void k_pose_keys(const int* __restrict__ e_ip, int eLocal, int numP, unsigned int* key, int* val)
{
	const int e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= eLocal) return;
	const int ip = e_ip[e] & 0x7fffffff;
	key[e] = ip < numP ? (unsigned)ip : (unsigned)numP;
	val[e] = e;
}

template <typename T>
__global__ void k_pose_stream(const int* __restrict__ src, const int* __restrict__ posePtr, int numP, int eLocal,
	const int* __restrict__ e_ip, const int* __restrict__ e_il,
	const T* __restrict__ mx, const T* __restrict__ my, const T* __restrict__ mz, const T* __restrict__ om,
	int* p_il, T* pmx, T* pmy, T* pmz, T* pom)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= eLocal || k >= posePtr[numP]) return;   // entries past posePtr[numP] belong to fixed poses
	const int e = src[k];
	p_il[k] = e_il[e] | (e_ip[e] & (int)0x80000000u);
	pmx[k] = mx[e]; pmy[k] = my[e]; pmz[k] = mz[e]; pom[k] = om[e];
}

// first column partner of Hpl block i: i itself, or -- when its pose observes the landmark through more than one edge (a
// repeated pair) -- the first of that pose's blocks in the column, so that the diagonal destination gets every ordered pair
__device__ __forceinline__ int first_partner(const int* __restrict__ hplRowInd, int colBeg, int i)
{
	int j = i;
	while (j > colBeg && hplRowInd[j - 1] == hplRowInd[i]) j--;
	return j;
}

// number of block products emitted by Hpl block i: its column partners j >= first_partner(i)
__global__ void k_prod_count(const int* __restrict__ hplLmG, const int* __restrict__ hplColPtr, const int* __restrict__ hplRowInd, int nhpl,
	int* cnt, Meta* meta)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= nhpl) return;
	const int l = hplLmG[i];
	const int j0 = first_partner(hplRowInd, hplColPtr[l], i);
	if (j0 < i) meta->repeats = 1;
	cnt[i] = hplColPtr[l + 1] - j0;
}

// products (i,j), j >= first_partner(i) in one landmark column, keyed by destination block (row_i,row_j); products of foreign
// landmarks (other ranks) keep their key (global pattern) but are marked pi = -1
__global__ void k_prod_emit(const int* __restrict__ hplLmG, const int* __restrict__ hplColPtr, const int* __restrict__ hplRowInd,
	const int* __restrict__ off, int nhpl, int lmBeg, int lmEnd, int hplBase, unsigned long long* pkey, int* pval, int* pi, int* pj)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= nhpl) return;
	const int l = hplLmG[i];
	const int cend = hplColPtr[l + 1];
	const bool local = l >= lmBeg && l < lmEnd;
	const unsigned long long hi = (unsigned long long)(unsigned)hplRowInd[i] << 32;
	int n = off[i];
	for (int j = first_partner(hplRowInd, hplColPtr[l], i); j < cend; j++, n++) {
		pkey[n] = hi | (unsigned)hplRowInd[j];
		pval[n] = n;
		pi[n] = local ? i - hplBase : -1;
		pj[n] = j - hplBase;
	}
}

// one dummy product per free pose so that every diagonal block exists
__global__ void k_prod_diag(int numP, long long nmul, unsigned long long* pkey, int* pval, int* pi, int* pj)
{
	const int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= numP) return;
	const long long n = nmul + p;
	pkey[n] = ((unsigned long long)(unsigned)p << 32) | (unsigned)p;
	pval[n] = (int)n; pi[n] = -1; pj[n] = -1;
}

__global__ void k_heads(const unsigned long long* __restrict__ keys, int n, int* head)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	head[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

__global__ void k_nblk(const int* __restrict__ head, const int* __restrict__ blkId, int n, Meta* meta)
{
	if (blockIdx.x == 0 && threadIdx.x == 0) meta->nblk = n > 0 ? blkId[n - 1] + head[n - 1] : 0;
}

__global__ void k_blocks(const unsigned long long* __restrict__ keys, const int* __restrict__ pvalSorted, const int* __restrict__ head,
	const int* __restrict__ blkId, const int* __restrict__ pi, const int* __restrict__ pj, int n,
	int* blkRow, int* blkCol, int* prodPtr, int* prodI, int* prodJ)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > n) return;
	if (i == n) { const int nb = n > 0 ? blkId[n - 1] + head[n - 1] : 0; prodPtr[nb] = n; return; }
	if (head[i]) { const int k = blkId[i]; blkRow[k] = (int)(keys[i] >> 32); blkCol[k] = (int)(keys[i] & 0xffffffffu); prodPtr[k] = i; }
	const int s = pvalSorted[i];
	prodI[i] = pi[s]; prodJ[i] = pj[s];
}

// ---- landmark-sharded runs: keep only this rank's products (and the diagonal placeholders) in the destination-sorted list ----
__global__ void k_local_flag(const int* __restrict__ prodI, const int* __restrict__ prodJ, int n, int* flag)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > n) return;
	flag[i] = (i < n && (prodI[i] >= 0 || prodJ[i] < 0)) ? 1 : 0;      // local product, or the placeholder of a diagonal block
}
__global__ void k_compact_products(const int* __restrict__ prodI, const int* __restrict__ prodJ, const int* __restrict__ flag, const int* __restrict__ pos,
	int n, int* outI, int* outJ)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n || !flag[i]) return;
	outI[pos[i]] = prodI[i]; outJ[pos[i]] = prodJ[i];
}
__global__ void k_remap_ptr(const int* __restrict__ pos, int nblk, int* prodPtr)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k > nblk) return;
	prodPtr[k] = pos[prodPtr[k]];
}

// rowPtr[a] = first block k with blkRow[k] >= a
__global__ void k_rowptr_from_rows(const int* __restrict__ rows, int n, int numP, int* rowPtr)
{
	const int a = blockIdx.x * blockDim.x + threadIdx.x;
	if (a > numP) return;
	int lo = 0, hi = n;
	while (lo < hi) { const int mid = (lo + hi) >> 1; if (rows[mid] < a) lo = mid + 1; else hi = mid; }
	rowPtr[a] = lo;
}

// symmetric-full BSR entries: (a,b,k) and, off the diagonal, (b,a,k) -- sorted afterwards by (row,col)
__global__ void k_full_entries(const int* __restrict__ blkRow, const int* __restrict__ blkCol, int nblk, int numP, unsigned long long* key, int* val)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= nblk) return;
	const unsigned a = (unsigned)blkRow[k], b = (unsigned)blkCol[k];
	key[2 * (size_t)k] = ((unsigned long long)a << 32) | b; val[2 * (size_t)k] = k << 1;
	// the unused second slot of a diagonal block sorts behind every real entry (row = numP)
	key[2 * (size_t)k + 1] = a == b ? ((unsigned long long)(unsigned)numP << 32) : (((unsigned long long)b << 32) | a);
	val[2 * (size_t)k + 1] = (k << 1) | 1;
}

__global__ void k_full_finish(const unsigned long long* __restrict__ key, const int* __restrict__ val, int nfull,
	const int* __restrict__ blkRow, const int* __restrict__ blkCol, int* fColInd, int* u2f, int* u2fT)
{
	const int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= nfull) return;
	fColInd[p] = (int)(key[p] & 0xffffffffu);
	const int k = val[p] >> 1;
	if (val[p] & 1) u2fT[k] = p;
	else { u2f[k] = p; if (blkRow[k] == blkCol[k]) u2fT[k] = p; }
}

inline int bits_for(unsigned long long maxValue)
{
	int b = 1;
	while (b < 64 && (maxValue >> b) != 0) b++;
	return b;
}

}  // namespace sgpu
}  // namespace cuba_b200
