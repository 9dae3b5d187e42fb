// cuba_peer_reduce.cuh -- all-reduce of the Schur matrix over NVLink peer memory, one kernel per GPU.
//
// Landmark-sharded runs sum the upper Hsc blocks and bsc of all ranks once per LM trial (66 MB of fp64 on the 10 M-edge
// graph).  With ncclAllReduce that collective was most of the Schur stage on 8 GPUs.  Here every
// GPU maps the others' buffers (cudaIpc) and runs ONE cooperative kernel:
//   signal "my partial sums are complete" to every peer, wait for theirs (flags in the peers' memory, system-scope fences);
//   reduce-scatter: this GPU adds its 1/world slice over all ranks, reading the peers' slices directly through NVLink, in
//     rank order 0..world-1 -- a fixed order, so every element is summed once, identically for everybody;
//   signal / wait again;
//   all-gather: copy the other slices from their owners.
// 2 x (world-1)/world of the buffer crosses NVLink per GPU, the minimum for an all-reduce; no staging copies, no NCCL call.
#pragma once

#include "cuba_pcg2.cuh"

namespace cuba_b200 {
namespace peer {

constexpr int MAXW = 8;
constexpr int BLOCK = 512;

template <typename T>
struct Args {
	T* local;                       // this rank's buffer (n elements, then the signal block)
	T* peers[MAXW];                 // the same buffer of every rank (own entry = local)
	unsigned int* sigLocal;         // [2][MAXW] signals written by the peers into this rank's memory
	unsigned int* sigPeer[MAXW];    // the signal block of every rank
	size_t n;
	int rank, world;
	unsigned int epoch;             // call counter, identical on every rank
	GridBar* bar;
};

__device__ __forceinline__ void st_sys_u32(unsigned int* p, unsigned int v) { asm volatile("st.volatile.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned int ld_sys_u32(const unsigned int* p) { unsigned int v; asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
template <typename T> struct Vec2;
template <> struct Vec2<double> { static __device__ __forceinline__ void ld(const double* p, double& a, double& b) { asm volatile("ld.volatile.global.v2.f64 {%0, %1}, [%2];" : "=d"(a), "=d"(b) : "l"(p) : "memory"); } };
template <> struct Vec2<float> { static __device__ __forceinline__ void ld(const float* p, float& a, float& b) { asm volatile("ld.volatile.global.v2.f32 {%0, %1}, [%2];" : "=f"(a), "=f"(b) : "l"(p) : "memory"); } };

// The CTAs of one rank: this CTA's index lc() among them and their number nctas().  k_peer_allreduce reads blockIdx.x and
// gridDim.x where it uses them (OneRank), k_peer_allreduce_ranks takes them from its rank's share of the grid (RankShare).
struct OneRank {
	__device__ __forceinline__ unsigned int lc() const { return blockIdx.x; }
	__device__ __forceinline__ unsigned int nctas() const { return gridDim.x; }
};
struct RankShare {
	unsigned int l, n;
	__device__ __forceinline__ unsigned int lc() const { return l; }
	__device__ __forceinline__ unsigned int nctas() const { return n; }
};

// every rank signals phase `ph` to all ranks and waits until all ranks have signalled it (CTA 0), then the rank's CTAs proceed
template <typename T, typename Ctas>
__device__ __forceinline__ void rank_barrier(const Args<T>& a, int ph, unsigned int& gen, const Ctas& g)
{
	if (g.lc() == 0 && threadIdx.x < a.world) {
		__threadfence_system();
		st_sys_u32(a.sigPeer[threadIdx.x] + ph * MAXW + a.rank, a.epoch);
		while ((int)(ld_sys_u32(a.sigLocal + ph * MAXW + threadIdx.x) - a.epoch) < 0) { }
		__threadfence_system();
	}
	grid_barrier(a.bar, g.nctas(), gen);
}

template <typename T, typename Ctas>
__device__ __forceinline__ void allreduce_body(const Args<T>& a, const Ctas& g)
{
	__shared__ unsigned int s_gen;
	if (threadIdx.x == 0) s_gen = ld_acquire_u32(&a.bar->gen);
	__syncthreads();
	unsigned int gen = s_gen;
	const size_t per = ((a.n + a.world - 1) / a.world + 1) & ~(size_t)1;      // slice length, even (two-element vector loads)
	const size_t stride = (size_t)g.nctas() * BLOCK * 2, first = ((size_t)g.lc() * BLOCK + threadIdx.x) * 2;
	rank_barrier(a, 0, gen, g);                                                     // everybody's partial sums are in place
	{
		const size_t lo = per * a.rank, hi = lo + per < a.n ? lo + per : a.n;
		for (size_t i = lo + first; i < hi; i += stride) {
			T s0 = T(0), s1 = T(0);
			const bool two = i + 1 < hi;
			for (int q = 0; q < a.world; q++) {
				T v0, v1 = T(0);
				if (two) Vec2<T>::ld(a.peers[q] + i, v0, v1);
				else v0 = *(volatile const T*)(a.peers[q] + i);
				s0 += v0; s1 += v1;
			}
			__stcg(a.local + i, s0);
			if (two) __stcg(a.local + i + 1, s1);
		}
	}
	grid_barrier(a.bar, g.nctas(), gen);
	rank_barrier(a, 1, gen, g);                                                     // every slice is reduced at its owner
	for (int q = 0; q < a.world; q++) {
		if (q == a.rank) continue;
		const size_t lo = per * q, hi = lo + per < a.n ? lo + per : a.n;
		for (size_t i = lo + first; i < hi; i += stride) {
			T v0, v1 = T(0);
			const bool two = i + 1 < hi;
			if (two) Vec2<T>::ld(a.peers[q] + i, v0, v1);
			else v0 = *(volatile const T*)(a.peers[q] + i);
			__stcg(a.local + i, v0);
			if (two) __stcg(a.local + i + 1, v1);
		}
	}
}

template <typename T>
__global__ void __launch_bounds__(BLOCK, 1) k_peer_allreduce(const Args<T> a) { allreduce_body(a, OneRank{}); }

// W ranks emulated on one GPU (cuba_debug_peer_allreduce): one cooperative launch of W * nctas CTAs, CTA b acting as CTA
// b % nctas of rank b / nctas with that rank's arguments (and GridBar) args[b / nctas]
template <typename T>
__global__ void __launch_bounds__(BLOCK, 1) k_peer_allreduce_ranks(const Args<T>* args, unsigned int nctas)
{
	allreduce_body(args[blockIdx.x / nctas], RankShare{ blockIdx.x % nctas, nctas });
}

}  // namespace peer
}  // namespace cuba_b200
