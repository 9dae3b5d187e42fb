// cuba_levels.cuh -- edge levels (g2o Edge::setLevel + initializeOptimization(0)) on the device.
//
// An edge at level 1 stays in the problem but is left out of the objective and the normal equations.  Its information value is
// zeroed in the three streams the J+H kernels read (landmark-major e_om, pose-major p_om, the warp-tile records of cuba_jh4.cuh):
// with a finite residual, omega = 0 contributes exact zeros to Hpp, bp, Hll, bl, Hpl, Hsc and chi2 under every robust kernel
// (rho(0) = 0), so neither the J+H, the Schur nor the PCG kernels know about levels.  The caller's omega stays in e_om0, the
// landmark-major copy the classification and the per-edge chi2 read.
//
//   k_classify_edges   one thread per local edge: the outlier test of ORB-SLAM2's local BA / pose optimisation on the committed
//                      estimate (chi2 against a threshold per edge type, optionally the depth), new level, four counts per block
//   k_sum_counts       one CTA: the block partials in a fixed order
//   k_mask_omega       e_om[k] = level ? 0 : e_om0[k]   (bit for bit what k_edge_stream writes for omega = 0)
//   k_pose_omega       the omega lane of the pose-major stream (k_pose_stream without the index lanes)
//   k_levels_out       a rank's levels into an edge-id-ordered fp64 array (summed over the ranks like the per-edge chi2)
// The warp-tile records are re-emitted with jh4::k_emit, as a structure-reuse set_problem does.
#pragma once

#include "cuba_kernels.cuh"

namespace cuba_b200 {
namespace lv {

constexpr int FAIL_DEPTH = 1;    // include/cuba_b200.h: CUBA_CLASSIFY_DEPTH
constexpr int REINCLUDE = 2;     // CUBA_CLASSIFY_REINCLUDE

// block partials: [block][4] = included mono, included stereo, newly excluded, re-included
template <typename T>
__global__ void __launch_bounds__(RED_BLOCK) k_classify_edges(const ChiArgs<T> a, const int* __restrict__ userId, unsigned char* level,
	double chi2Mono, double chi2Stereo, int flags, int* partial)
{
	__shared__ int s_cnt[RED_BLOCK / 32][4];
	const int e = blockIdx.x * RED_BLOCK + threadIdx.x;
	int c[4] = { 0, 0, 0, 0 };
	if (e < a.E) {
		const int ipf = a.ip[e];
		const bool stereo = ipf < 0;
		T q[4], t[3], cm[5], X[3], m[3], Xc[3], r[3];
		load_pose(a.pose, a.cam, ipf & 0x7fffffff, q, t, cm);
		load_xw(a.Xw, a.il[e], X);
		m[0] = a.mx[e]; m[1] = a.my[e]; m[2] = stereo ? a.mz[e] : T(0);
		edge_residual(q, t, cm, X, m, stereo, Xc, r);
		// the value k_chi_sqs reports for this edge
		const double chi2 = (double)(a.om[e] * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]));
		const bool fail = chi2 > (stereo ? chi2Stereo : chi2Mono) || ((flags & FAIL_DEPTH) && Xc[2] <= T(0));
		const int u = userId[e];
		const int old = level[u];
		const int now = (flags & REINCLUDE) ? (fail ? 1 : 0) : (old | (fail ? 1 : 0));
		if (now != old) level[u] = (unsigned char)now;
		c[0] = !now && !stereo; c[1] = !now && stereo; c[2] = !old && now; c[3] = old && !now;
	}
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
	for (int k = 0; k < 4; k++) {
		int v = c[k];
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
		if (lane == 0) s_cnt[w][k] = v;
	}
	__syncthreads();
	if (threadIdx.x < 4) {
		int s = 0;
		for (int i = 0; i < RED_BLOCK / 32; i++) s += s_cnt[i][threadIdx.x];
		partial[4 * (size_t)blockIdx.x + threadIdx.x] = s;
	}
}

// out[k] = sum over the n blocks of partial[.][k], k < 4 (single CTA; integer sums, written as fp64 for the all-reduce)
__global__ void __launch_bounds__(RED_BLOCK) k_sum_counts(const int* __restrict__ partial, int n, double* out)
{
	__shared__ long long s_red[RED_BLOCK / 32];
	for (int k = 0; k < 4; k++) {
		long long s = 0;
		for (int i = threadIdx.x; i < n; i += RED_BLOCK) s += partial[4 * (size_t)i + k];
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
		if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = s;
		__syncthreads();
		if (threadIdx.x == 0) {
			long long tot = 0;
			for (int i = 0; i < RED_BLOCK / 32; i++) tot += s_red[i];
			out[k] = (double)tot;
		}
		__syncthreads();
	}
}

template <typename T>
__global__ void k_mask_omega(const T* __restrict__ om0, const int* __restrict__ userId, const unsigned char* __restrict__ level, int eLocal, T* om)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= eLocal) return;
	om[k] = level[userId[k]] ? T(0) : om0[k];
}

template <typename T>
__global__ void k_pose_omega(const int* __restrict__ src, const int* __restrict__ posePtr, int numP, int eLocal, const T* __restrict__ om, T* pom)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= eLocal || k >= posePtr[numP]) return;   // entries past posePtr[numP] belong to fixed poses
	pom[k] = om[src[k]];
}

__global__ void k_levels_out(const int* __restrict__ userId, const unsigned char* __restrict__ level, int eLocal, double* out)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= eLocal) return;
	const int u = userId[k];
	out[u] = (double)level[u];
}

}  // namespace lv
}  // namespace cuba_b200
