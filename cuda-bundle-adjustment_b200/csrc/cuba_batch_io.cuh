// cuba_batch_io.cuh -- the packed layouts of the batched LM kernels (k_pose_batch, k_sim3_batch, k_point_batch) and the kernels that
// validate, pack and unpack a batch whose arrays are already in device memory (cuba_engine_optimize_poses_device / _sim3_device /
// _points_device).
//
// PoseLayout, Sim3Layout and PointLayout are the one definition of the packed records: the host round trip (Engine::optimize_poses /
// optimize_sim3 / optimize_points) packs into them, the device path packs into them, and cuba_*_batch_workspace_bytes sizes them.  The records are
// those the LM kernels read: an input area (nIn doubles) followed, in the device path's workspace, by the results (nOut doubles).
//
// The device path runs, on one stream:
//   1. status = 0, then k_validate_*: the host entry points' data checks, OR-ed into the status word (CUBA_BATCH_* bits);
//   2. k_pack_*: copies the caller's arrays into the input records, one thread per scalar, with no arithmetic, so the packed bytes
//      equal the host loop's (signed zeros and NaN payloads included).  With status != 0 it writes every CSR pointer as 0 instead:
//      the LM kernel, which does not read the status, then sees B empty problems and writes only into the workspace;
//   3. the unchanged LM kernel on the workspace;
//   4. k_unpack_*: with status == 0, copies the results into the caller's arrays in the host entry points' layouts.
#pragma once

#include "cuba_pose_batch.cuh"
#include "cuba_sim3_batch.cuh"
#include "cuba_point_batch.cuh"

namespace cuba_b200 {
namespace bio {

// pose batch, in doubles.  input: pose [B][8] | cam [B][8] | edges [E][8] | ptr2, ptr3 as int32 [B+1] each.  results: pose [B][8] |
// stats [nStat] (4 doubles each) | counts [B][R][4], nstats [B][R] as int32 | levels [E] bytes
struct PoseLayout {
	size_t oCam, oEdge, oPtr, nIn;
	size_t oStat, oInt, oLev, nOut;
	__host__ __device__ PoseLayout(size_t B, size_t E, size_t R, size_t nStat)
	{
		oCam = 8 * B; oEdge = 16 * B; oPtr = oEdge + 8 * E; nIn = oPtr + (B + 1);
		oStat = 8 * B; oInt = oStat + 4 * nStat; oLev = oInt + (5 * B * R + 1) / 2; nOut = oLev + (E + 7) / 8;
	}
};

// Sim3 batch, in doubles.  input: problems [B][PROB] | pairs [N][PAIR] | ptr as int32 [B+1].  results: S [B][8] | stats [nStat]
// (4 doubles each) | ninliers [B], nstats [B][2] as int32 | levels [N] bytes
struct Sim3Layout {
	size_t oPair, oPtr, nIn;
	size_t oStat, oInt, oLev, nOut;
	__host__ __device__ Sim3Layout(size_t B, size_t N, size_t nStat)
	{
		oPair = s3::PROB * B; oPtr = oPair + s3::PAIR * N; nIn = oPtr + (B + 2) / 2;
		oStat = 8 * B; oInt = oStat + 4 * nStat; oLev = oInt + (3 * B + 1) / 2; nOut = oLev + (N + 7) / 8;
	}
};

// point batch, in doubles.  input: Xw [B][4] | pose [P][8] | cam [P][8] | edges [E][4] | iP [E], ptr2, ptr3 [B+1] each as int32.
// results: Xw [B][4] | stats [nStat] (4 doubles each) | counts [B][R][4], nstats [B][R] as int32 | levels [E] bytes
struct PointLayout {
	size_t oPose, oCam, oEdge, oIdx, nIn;
	size_t oStat, oInt, oLev, nOut;
	__host__ __device__ PointLayout(size_t B, size_t P, size_t E, size_t R, size_t nStat)
	{
		oPose = 4 * B; oCam = oPose + 8 * P; oEdge = oCam + 8 * P; oIdx = oEdge + 4 * E; nIn = oIdx + (E + 2 * (B + 1) + 1) / 2;
		oStat = 4 * B; oInt = oStat + 4 * nStat; oLev = oInt + (5 * B * R + 1) / 2; nOut = oLev + (E + 7) / 8;
	}
};

constexpr int BLOCK = 256;
constexpr unsigned MAX_GRID = 4096;   // the grid-stride kernels
constexpr int POINTS_PER_BLOCK = BLOCK / 32;   // k_pack_points / k_unpack_points: one warp per point

__device__ __forceinline__ size_t gtid() { return (size_t)blockIdx.x * blockDim.x + threadIdx.x; }
__device__ __forceinline__ size_t gstride() { return (size_t)gridDim.x * blockDim.x; }

// the checks of csr_ok on entry i of ptr[B+1]
__device__ __forceinline__ int ptr_bits(const int32_t* ptr, int B, int count, size_t i)
{
	int bad = 0;
	if (i == 0 && ptr[0] != 0) bad |= CUBA_BATCH_PTR_START;
	if (i < (size_t)B && ptr[i + 1] < ptr[i]) bad |= CUBA_BATCH_PTR_DECREASES;
	if (i == (size_t)B && ptr[B] != count) bad |= CUBA_BATCH_PTR_END;
	return bad;
}

__device__ __forceinline__ int finite_bits(const double* p, size_t n, int bit)
{
	for (size_t i = gtid(); i < n; i += gstride())
		if (!isfinite(p[i])) return bit;
	return 0;
}

// every thread of the grid calls this once, at the end
__device__ __forceinline__ void report(int bad, int32_t* status)
{
	bad = __reduce_or_sync(0xffffffffu, bad);
	if ((threadIdx.x & 31) == 0 && bad) atomicOr(status, bad);
}

__global__ void __launch_bounds__(BLOCK) k_validate_poses(const cuba_pose_batch bt, int32_t* status)
{
	int bad = 0;
	for (size_t i = gtid(); i <= (size_t)bt.B; i += gstride()) bad |= ptr_bits(bt.ptr2, bt.B, bt.E2, i) | ptr_bits(bt.ptr3, bt.B, bt.E3, i);
	bad |= finite_bits(bt.omega2, (size_t)bt.E2, CUBA_BATCH_NONFINITE_ITEM) | finite_bits(bt.omega3, (size_t)bt.E3, CUBA_BATCH_NONFINITE_ITEM);
	report(bad, status);
}

__global__ void __launch_bounds__(BLOCK) k_validate_sim3(const cuba_sim3_batch bt, int32_t* status)
{
	const size_t B = (size_t)bt.B, N = (size_t)bt.N;
	int bad = 0;
	for (size_t i = gtid(); i <= B; i += gstride()) bad |= ptr_bits(bt.ptr, bt.B, bt.N, i);
	for (size_t b = gtid(); b < B; b += gstride())
		if (isfinite(bt.s[b]) && !(bt.s[b] > 0)) bad |= CUBA_BATCH_SCALE;
	constexpr int P = CUBA_BATCH_NONFINITE_PROBLEM, I = CUBA_BATCH_NONFINITE_ITEM;
	bad |= finite_bits(bt.q, 4 * B, P) | finite_bits(bt.t, 3 * B, P) | finite_bits(bt.s, B, P) | finite_bits(bt.cam1, 4 * B, P) |
		finite_bits(bt.cam2, 4 * B, P);
	bad |= finite_bits(bt.X1, 3 * N, I) | finite_bits(bt.X2, 3 * N, I) | finite_bits(bt.obs1, 2 * N, I) | finite_bits(bt.obs2, 2 * N, I) |
		finite_bits(bt.omega1, N, I) | finite_bits(bt.omega2, N, I);
	report(bad, status);
}

// one CTA per frame: the records of Engine::optimize_poses' host loop; a frame's mono edge i at ptr3[b] + i, its stereo edge j at
// ptr2[b+1] + j
__global__ void __launch_bounds__(BLOCK) k_pack_poses(const cuba_pose_batch bt, const PoseLayout L, double* in, const int32_t* status)
{
	const int B = bt.B, b = blockIdx.x, tid = threadIdx.x;
	int32_t* p2 = (int32_t*)(in + L.oPtr);
	int32_t* p3 = p2 + B + 1;
	const bool ok = *status == 0;
	if (tid == 0) {
		p2[b] = ok ? bt.ptr2[b] : 0; p3[b] = ok ? bt.ptr3[b] : 0;
		if (b == B - 1) { p2[B] = ok ? bt.ptr2[B] : 0; p3[B] = ok ? bt.ptr3[B] : 0; }
	}
	if (!ok) return;
	if (tid < 8) {
		in[8 * (size_t)b + tid] = tid < 4 ? bt.q[4 * (size_t)b + tid] : tid < 7 ? bt.t[3 * (size_t)b + tid - 4] : 0.0;
		in[L.oCam + 8 * (size_t)b + tid] = tid < 5 ? bt.cam[5 * (size_t)b + tid] : 0.0;
	}
	const size_t i0 = (size_t)bt.ptr2[b], n2 = (size_t)bt.ptr2[b + 1] - i0, j0 = (size_t)bt.ptr3[b], n3 = (size_t)bt.ptr3[b + 1] - j0;
	double* em = in + L.oEdge + 8 * (j0 + i0);
	for (size_t k = tid; k < 8 * n2; k += BLOCK) {
		const size_t i = i0 + k / 8;
		const int c = (int)(k & 7);
		em[k] = c < 3 ? bt.X2[3 * i + c] : c < 5 ? bt.meas2[2 * i + c - 3] : c == 6 ? bt.omega2[i] : 0.0;
	}
	double* es = in + L.oEdge + 8 * ((size_t)bt.ptr2[b + 1] + j0);
	for (size_t k = tid; k < 8 * n3; k += BLOCK) {
		const size_t j = j0 + k / 8;
		const int c = (int)(k & 7);
		es[k] = c < 3 ? bt.X3[3 * j + c] : c < 6 ? bt.meas3[3 * j + c - 3] : c == 6 ? bt.omega3[j] : 0.0;
	}
}

// one CTA per frame: q, t, stats, counts, nstats and the levels back in mono-then-stereo order.  statPer: stat slots per frame
__global__ void __launch_bounds__(BLOCK) k_unpack_poses(const PoseLayout L, int B, int R, int E2, int statPer, const double* in,
	double* qOut, double* tOut, uint8_t* levelsOut, int32_t* counts, cuba_iter_stat* stats, int32_t* nstats, const int32_t* status)
{
	if (*status) return;
	const int b = blockIdx.x, tid = threadIdx.x;
	const double* o = in + L.nIn;
	if (tid < 4) qOut[4 * (size_t)b + tid] = o[8 * (size_t)b + tid];
	else if (tid < 7) tOut[3 * (size_t)b + tid - 4] = o[8 * (size_t)b + tid];
	if (stats) {
		const size_t n = 4 * (size_t)statPer, k0 = n * b;
		const unsigned long long* s = (const unsigned long long*)(o + L.oStat);
		unsigned long long* d = (unsigned long long*)stats;
		for (size_t k = tid; k < n; k += BLOCK) d[k0 + k] = s[k0 + k];
	}
	const int32_t* oi = (const int32_t*)(o + L.oInt);
	if (counts)
		for (int k = tid; k < 4 * R; k += BLOCK) counts[(size_t)b * 4 * R + k] = oi[(size_t)b * 4 * R + k];
	if (nstats)
		for (int k = tid; k < R; k += BLOCK) nstats[(size_t)b * R + k] = oi[4 * (size_t)B * R + (size_t)b * R + k];
	if (levelsOut) {
		const int32_t* p2 = (const int32_t*)(in + L.oPtr);
		const int32_t* p3 = p2 + B + 1;
		const uint8_t* lv = (const uint8_t*)(o + L.oLev);
		for (size_t i = (size_t)p2[b] + tid; i < (size_t)p2[b + 1]; i += BLOCK) levelsOut[i] = lv[(size_t)p3[b] + i];
		for (size_t j = (size_t)p3[b] + tid; j < (size_t)p3[b + 1]; j += BLOCK) levelsOut[(size_t)E2 + j] = lv[(size_t)p2[b + 1] + j];
	}
}

// grid-stride over the problem records, the pair records and ptr: the records of Engine::optimize_sim3's host loop
__global__ void __launch_bounds__(BLOCK) k_pack_sim3(const cuba_sim3_batch bt, const Sim3Layout L, double* in, const int32_t* status)
{
	const size_t B = (size_t)bt.B, nP = s3::PROB * B, nQ = s3::PAIR * (size_t)bt.N, total = nP + nQ + B + 1;
	const bool ok = *status == 0;
	int32_t* ptr = (int32_t*)(in + L.oPtr);
	for (size_t k = gtid(); k < total; k += gstride()) {
		if (k >= nP + nQ) {
			ptr[k - nP - nQ] = ok ? bt.ptr[k - nP - nQ] : 0;
		} else if (!ok) {
			continue;
		} else if (k < nP) {
			const size_t b = k / s3::PROB;
			const int c = (int)(k % s3::PROB);
			in[k] = c < 4 ? bt.q[4 * b + c] : c < 7 ? bt.t[3 * b + c - 4] : c == 7 ? bt.s[b] : c < 12 ? bt.cam1[4 * b + c - 8] :
				c < 16 ? bt.cam2[4 * b + c - 12] : c == 16 ? (bt.fix_scale && bt.fix_scale[b] ? 1.0 : 0.0) : 0.0;
		} else {
			const size_t i = (k - nP) / s3::PAIR;
			const int c = (int)((k - nP) % s3::PAIR);
			in[k] = c < 3 ? bt.X1[3 * i + c] : c < 6 ? bt.X2[3 * i + c - 3] : c < 8 ? bt.obs1[2 * i + c - 6] : c < 10 ? bt.obs2[2 * i + c - 8] :
				c == 10 ? bt.omega1[i] : bt.omega2[i];
		}
	}
}

// grid-stride over S, stats, ninliers, nstats and levels.  nStat: stat slots of the whole batch (0 without stats)
__global__ void __launch_bounds__(BLOCK) k_unpack_sim3(const Sim3Layout L, int Bi, int Ni, size_t nStat, const double* in, double* qOut,
	double* tOut, double* sOut, uint8_t* levelsOut, int32_t* ninliers, cuba_iter_stat* stats, int32_t* nstats, const int32_t* status)
{
	if (*status) return;
	const size_t B = (size_t)Bi, N = (size_t)Ni;
	const double* o = in + L.nIn;
	for (size_t k = gtid(); k < 8 * B; k += gstride()) {
		const size_t b = k / 8;
		const int c = (int)(k % 8);
		if (c < 4) qOut[4 * b + c] = o[k];
		else if (c < 7) tOut[3 * b + c - 4] = o[k];
		else sOut[b] = o[k];
	}
	if (stats) {
		const unsigned long long* s = (const unsigned long long*)(o + L.oStat);
		for (size_t k = gtid(); k < 4 * nStat; k += gstride()) ((unsigned long long*)stats)[k] = s[k];
	}
	const int32_t* oi = (const int32_t*)(o + L.oInt);
	if (ninliers)
		for (size_t k = gtid(); k < B; k += gstride()) ninliers[k] = oi[k];
	if (nstats)
		for (size_t k = gtid(); k < 2 * B; k += gstride()) nstats[k] = oi[B + k];
	if (levelsOut) {
		const uint8_t* lv = (const uint8_t*)(o + L.oLev);
		for (size_t k = gtid(); k < N; k += gstride()) levelsOut[k] = lv[k];
	}
}

__global__ void __launch_bounds__(BLOCK) k_validate_points(const cuba_point_batch bt, int32_t* status)
{
	int bad = 0;
	for (size_t i = gtid(); i <= (size_t)bt.B; i += gstride()) bad |= ptr_bits(bt.ptr2, bt.B, bt.E2, i) | ptr_bits(bt.ptr3, bt.B, bt.E3, i);
	bad |= finite_bits(bt.omega2, (size_t)bt.E2, CUBA_BATCH_NONFINITE_ITEM) | finite_bits(bt.omega3, (size_t)bt.E3, CUBA_BATCH_NONFINITE_ITEM);
	for (size_t i = gtid(); i < (size_t)bt.E2; i += gstride())
		if (bt.iP2[i] < 0 || bt.iP2[i] >= bt.P) bad |= CUBA_BATCH_INDEX;
	for (size_t i = gtid(); i < (size_t)bt.E3; i += gstride())
		if (bt.iP3[i] < 0 || bt.iP3[i] >= bt.P) bad |= CUBA_BATCH_INDEX;
	report(bad, status);
}

// one warp per point, and the pose table grid-stride: the records of Engine::optimize_points' host loop; a point's mono edge i at
// ptr3[b] + i, its stereo edge j at ptr2[b+1] + j
__global__ void __launch_bounds__(BLOCK) k_pack_points(const cuba_point_batch bt, const PointLayout L, double* in, const int32_t* status)
{
	const int B = bt.B, b = blockIdx.x * POINTS_PER_BLOCK + (threadIdx.x >> 5), lane = threadIdx.x & 31;
	int32_t* ip = (int32_t*)(in + L.oIdx);
	const size_t E = (size_t)bt.E2 + (size_t)bt.E3;
	int32_t* p2 = ip + E;
	int32_t* p3 = p2 + B + 1;
	const bool ok = *status == 0;
	if (b < B && lane == 0) {
		p2[b] = ok ? bt.ptr2[b] : 0; p3[b] = ok ? bt.ptr3[b] : 0;
		if (b == B - 1) { p2[B] = ok ? bt.ptr2[B] : 0; p3[B] = ok ? bt.ptr3[B] : 0; }
	}
	if (!ok) return;
	const size_t P = (size_t)bt.P;
	for (size_t k = gtid(); k < 16 * P; k += gstride()) {
		const size_t p = (k % (8 * P)) / 8;
		const int c = (int)(k & 7);
		in[L.oPose + k] = k < 8 * P ? (c < 4 ? bt.q[4 * p + c] : c < 7 ? bt.t[3 * p + c - 4] : 0.0) : (c < 5 ? bt.cam[5 * p + c] : 0.0);
	}
	if (b >= B) return;
	if (lane < 4) in[4 * (size_t)b + lane] = lane < 3 ? bt.Xw[3 * (size_t)b + lane] : 0.0;
	const size_t i0 = (size_t)bt.ptr2[b], n2 = (size_t)bt.ptr2[b + 1] - i0, j0 = (size_t)bt.ptr3[b], n3 = (size_t)bt.ptr3[b + 1] - j0;
	const size_t m0 = i0 + j0, s0 = (size_t)bt.ptr2[b + 1] + j0;
	for (size_t k = lane; k < 4 * n2; k += 32) {
		const size_t i = i0 + k / 4;
		const int c = (int)(k & 3);
		in[L.oEdge + 4 * m0 + k] = c < 2 ? bt.meas2[2 * i + c] : c == 3 ? bt.omega2[i] : 0.0;
	}
	for (size_t k = lane; k < n2; k += 32) ip[m0 + k] = bt.iP2[i0 + k];
	for (size_t k = lane; k < 4 * n3; k += 32) {
		const size_t j = j0 + k / 4;
		const int c = (int)(k & 3);
		in[L.oEdge + 4 * s0 + k] = c < 3 ? bt.meas3[3 * j + c] : bt.omega3[j];
	}
	for (size_t k = lane; k < n3; k += 32) ip[s0 + k] = bt.iP3[j0 + k];
}

// one warp per point: Xw, stats, counts, nstats and the levels back in mono-then-stereo order.  statPer: stat slots per point
__global__ void __launch_bounds__(BLOCK) k_unpack_points(const PointLayout L, int B, int R, int E2, int E3, int statPer, const double* in,
	double* XwOut, uint8_t* levelsOut, int32_t* counts, cuba_iter_stat* stats, int32_t* nstats, const int32_t* status)
{
	if (*status) return;
	const int b = blockIdx.x * POINTS_PER_BLOCK + (threadIdx.x >> 5), lane = threadIdx.x & 31;
	if (b >= B) return;
	const double* o = in + L.nIn;
	if (lane < 3) XwOut[3 * (size_t)b + lane] = o[4 * (size_t)b + lane];
	if (stats) {
		const size_t n = 4 * (size_t)statPer, k0 = n * b;
		const unsigned long long* s = (const unsigned long long*)(o + L.oStat);
		unsigned long long* d = (unsigned long long*)stats;
		for (size_t k = lane; k < n; k += 32) d[k0 + k] = s[k0 + k];
	}
	const int32_t* oi = (const int32_t*)(o + L.oInt);
	if (counts)
		for (int k = lane; k < 4 * R; k += 32) counts[(size_t)b * 4 * R + k] = oi[(size_t)b * 4 * R + k];
	if (nstats)
		for (int k = lane; k < R; k += 32) nstats[(size_t)b * R + k] = oi[4 * (size_t)B * R + (size_t)b * R + k];
	if (levelsOut) {
		const int32_t* p2 = (const int32_t*)(in + L.oIdx) + (size_t)E2 + (size_t)E3;
		const int32_t* p3 = p2 + B + 1;
		const uint8_t* lv = (const uint8_t*)(o + L.oLev);
		for (size_t i = (size_t)p2[b] + lane; i < (size_t)p2[b + 1]; i += 32) levelsOut[i] = lv[(size_t)p3[b] + i];
		for (size_t j = (size_t)p3[b] + lane; j < (size_t)p3[b + 1]; j += 32) levelsOut[(size_t)E2 + j] = lv[(size_t)p2[b + 1] + j];
	}
}

inline unsigned grid_for(size_t n) { return (unsigned)std::max<size_t>(1, std::min<size_t>(MAX_GRID, (n + BLOCK - 1) / BLOCK)); }

}  // namespace bio
}  // namespace cuba_b200
