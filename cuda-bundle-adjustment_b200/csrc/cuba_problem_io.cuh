// cuba_problem_io.cuh -- the engine's own problem on device-resident arrays (include/cuba_b200.h: cuba_engine_set_problem_device
// and the other *_device entry points of the engine's problem).  The caller's arrays are read and written where they are; these
// kernels only copy, compare and count, so every result is bit for bit that of the host entry point of the same name.
//
//   k_idx_differ     one thread per index word: *flag = 1 where a (iP, iL) list differs from the held problem's g_idx2 / g_idx3
//                    (the structure-reuse test of a set_problem whose lists the host cannot memcmp)
//   k_unpack_state   one thread per pose / landmark: the padded state records into the caller's flat q [4P], t [3P], Xw [3L], widened
//                    to fp64 as get_state does; a NULL output is skipped
//   k_levels_in      one thread per edge: level = (in != 0) (in == NULL: every level 0); per block, the edges at level 0 among all
//                    edges and among this rank's own (userId over eLocal), as partials 0 and 1 of lv::k_sum_counts
//   k_levels_narrow  an edge-id-ordered fp64 level array (lv::k_levels_out, summed over the ranks) to bytes
#pragma once

#include "cuba_kernels.cuh"

namespace cuba_b200 {
namespace pio {

__global__ void k_idx_differ(const int* __restrict__ a2, const int* __restrict__ b2, long long n2, const int* __restrict__ a3,
	const int* __restrict__ b3, long long n3, int* flag)
{
	const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
	const bool differ = i < n2 ? a2[i] != b2[i] : (i < n2 + n3 && a3[i - n2] != b3[i - n2]);
	if (differ) *flag = 1;
}

template <typename T>
__global__ void k_unpack_state(const T* __restrict__ pose, const T* __restrict__ Xw, int Pall, int Lall, double* q, double* t, double* X)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < Pall) {
		if (q) for (int k = 0; k < 4; k++) q[4 * (size_t)i + k] = (double)pose[8 * (size_t)i + k];
		if (t) for (int k = 0; k < 3; k++) t[3 * (size_t)i + k] = (double)pose[8 * (size_t)i + 4 + k];
	}
	if (i < Lall && X)
		for (int k = 0; k < 3; k++) X[3 * (size_t)i + k] = (double)Xw[4 * (size_t)i + k];
}

// partial[block][4] = edges at level 0 of all E, of the eLocal own edges, 0, 0
__global__ void __launch_bounds__(RED_BLOCK) k_levels_in(const unsigned char* __restrict__ in, int E, const int* __restrict__ userId, int eLocal,
	unsigned char* level, int* partial)
{
	__shared__ int s_cnt[RED_BLOCK / 32][2];
	const int i = blockIdx.x * RED_BLOCK + threadIdx.x;
	int c[2] = { 0, 0 };
	if (i < E) {
		const unsigned char v = in && in[i] != 0;
		level[i] = v;
		c[0] = !v;
	}
	if (i < eLocal) c[1] = !(in && in[userId[i]] != 0);
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
	for (int k = 0; k < 2; k++) {
		int v = c[k];
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
		if (lane == 0) s_cnt[w][k] = v;
	}
	__syncthreads();
	if (threadIdx.x < 4) {
		int s = 0;
		if (threadIdx.x < 2)
			for (int j = 0; j < RED_BLOCK / 32; j++) s += s_cnt[j][threadIdx.x];
		partial[4 * (size_t)blockIdx.x + threadIdx.x] = s;
	}
}

__global__ void k_levels_narrow(const double* __restrict__ in, int E, unsigned char* out)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < E) out[i] = in[i] != 0.0;
}

}  // namespace pio
}  // namespace cuba_b200
