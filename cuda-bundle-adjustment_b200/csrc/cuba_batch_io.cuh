// cuba_batch_io.cuh -- the packed layouts and records of the batched LM kernels (k_pose_batch, k_sim3_batch, k_point_batch), their
// packers, launchers and unpackers: on the host for cuba_engine_optimize_poses / _sim3 / _points, and as kernels that also validate
// the batch for cuba_engine_optimize_poses_device / _sim3_device / _points_device, whose arrays are already in device memory.
//
// PoseLayout, Sim3Layout and PointLayout are the one definition of where the packed records go, and the *_rec functions of what each
// record holds: both packers use them, and cuba_*_batch_workspace_bytes sizes the layouts.  The records are those the LM kernels
// read: an input area (nIn doubles) followed, in the device path's workspace, by the results (nOut doubles).
//
// The host path packs on the host, copies up, runs launch_*, copies down, synchronises and unpacks on the host.  The device path runs,
// on one stream:
//   1. status = 0, then k_validate_*: the host entry points' data checks, OR-ed into the status word (CUBA_BATCH_* bits);
//   2. k_pack_*: copies the caller's arrays into the input records, one thread per scalar, with no arithmetic, so the packed bytes
//      equal the host packer's (signed zeros and NaN payloads included).  With status != 0 it writes every CSR pointer as 0 instead:
//      the LM kernel, which does not read the status, then sees B empty problems and writes only into the workspace;
//   3. launch_*: the unchanged LM kernel on the workspace;
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

// ---- the records: scalar c of record i, from the caller's arrays -------------------------------------------------------------------

// pose [8]: q(4) t(3) pad -- a frame of the pose batch, a pose of the point batch's table
CUBA_HD double pose_rec(const double* q, const double* t, size_t i, int c) { return c < 4 ? q[4 * i + c] : c < 7 ? t[3 * i + c - 4] : 0.0; }
// camera [8]: fx fy cx cy bf pad
CUBA_HD double cam_rec(const double* cam, size_t i, int c) { return c < 5 ? cam[5 * i + c] : 0.0; }
// pose-batch edges [8]: X(3) meas(3) omega pad; a mono edge's meas[2] is 0
CUBA_HD double pose_mono_rec(const cuba_pose_batch& bt, size_t i, int c)
{
	return c < 3 ? bt.X2[3 * i + c] : c < 5 ? bt.meas2[2 * i + c - 3] : c == 6 ? bt.omega2[i] : 0.0;
}
CUBA_HD double pose_stereo_rec(const cuba_pose_batch& bt, size_t j, int c)
{
	return c < 3 ? bt.X3[3 * j + c] : c < 6 ? bt.meas3[3 * j + c - 3] : c == 6 ? bt.omega3[j] : 0.0;
}
// Sim3 problem [s3::PROB]: q(4) t(3) s cam1(4) cam2(4) fix_scale pad(3)
CUBA_HD double sim3_prob_rec(const cuba_sim3_batch& bt, size_t b, int c)
{
	return c < 4 ? bt.q[4 * b + c] : c < 7 ? bt.t[3 * b + c - 4] : c == 7 ? bt.s[b] : c < 12 ? bt.cam1[4 * b + c - 8] :
		c < 16 ? bt.cam2[4 * b + c - 12] : c == 16 ? (bt.fix_scale && bt.fix_scale[b] ? 1.0 : 0.0) : 0.0;
}
// Sim3 pair [s3::PAIR]: X1(3) X2(3) obs1(2) obs2(2) omega1 omega2
CUBA_HD double sim3_pair_rec(const cuba_sim3_batch& bt, size_t i, int c)
{
	return c < 3 ? bt.X1[3 * i + c] : c < 6 ? bt.X2[3 * i + c - 3] : c < 8 ? bt.obs1[2 * i + c - 6] : c < 10 ? bt.obs2[2 * i + c - 8] :
		c == 10 ? bt.omega1[i] : bt.omega2[i];
}
// point [4]: X(3) pad
CUBA_HD double point_rec(const cuba_point_batch& bt, size_t b, int c) { return c < 3 ? bt.Xw[3 * b + c] : 0.0; }
// point-batch edges [4]: meas(3) omega; a mono edge's meas[2] is 0
CUBA_HD double point_mono_rec(const cuba_point_batch& bt, size_t i, int c) { return c < 2 ? bt.meas2[2 * i + c] : c == 3 ? bt.omega2[i] : 0.0; }
CUBA_HD double point_stereo_rec(const cuba_point_batch& bt, size_t j, int c) { return c < 3 ? bt.meas3[3 * j + c] : bt.omega3[j]; }

// The packed slot of an edge of the pose and point batches: a problem's edges are contiguous, its mono edges first, so mono edge i
// of problem b sits at ptr3[b] + i and stereo edge j at ptr2[b+1] + j
CUBA_HD size_t edge_slot(const int32_t* ptr2, const int32_t* ptr3, size_t b, size_t i, bool stereo)
{
	return stereo ? (size_t)ptr2[b + 1] + i : (size_t)ptr3[b] + i;
}

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

// one CTA per frame
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
		in[8 * (size_t)b + tid] = pose_rec(bt.q, bt.t, b, tid);
		in[L.oCam + 8 * (size_t)b + tid] = cam_rec(bt.cam, b, tid);
	}
	const size_t i0 = (size_t)bt.ptr2[b], n2 = (size_t)bt.ptr2[b + 1] - i0, j0 = (size_t)bt.ptr3[b], n3 = (size_t)bt.ptr3[b + 1] - j0;
	double* em = in + L.oEdge + 8 * edge_slot(bt.ptr2, bt.ptr3, b, i0, false);
	for (size_t k = tid; k < 8 * n2; k += BLOCK) em[k] = pose_mono_rec(bt, i0 + k / 8, (int)(k & 7));
	double* es = in + L.oEdge + 8 * edge_slot(bt.ptr2, bt.ptr3, b, j0, true);
	for (size_t k = tid; k < 8 * n3; k += BLOCK) es[k] = pose_stereo_rec(bt, j0 + k / 8, (int)(k & 7));
}

// The results of problem b of a pose or point batch after its position, by threads `lane` of `step` (the host entries: 0 of 1): stats,
// counts, nstats and the levels back in mono-then-stereo order.  o: the packed results; p2: the packed ptr2, followed by ptr3
template <class Layout>
CUBA_HD void unpack_rounds(const Layout& L, const double* o, const int32_t* p2, int b, int B, int R, int E2, int statPer,
	int lane, int step, uint8_t* levelsOut, int32_t* counts, cuba_iter_stat* stats, int32_t* nstats)
{
	if (stats) {
		const size_t n = 4 * (size_t)statPer, k0 = n * b;
		const unsigned long long* s = (const unsigned long long*)(o + L.oStat);
		unsigned long long* d = (unsigned long long*)stats;
		for (size_t k = lane; k < n; k += step) d[k0 + k] = s[k0 + k];
	}
	const int32_t* oi = (const int32_t*)(o + L.oInt);
	if (counts)
		for (int k = lane; k < 4 * R; k += step) counts[(size_t)b * 4 * R + k] = oi[(size_t)b * 4 * R + k];
	if (nstats)
		for (int k = lane; k < R; k += step) nstats[(size_t)b * R + k] = oi[4 * (size_t)B * R + (size_t)b * R + k];
	if (levelsOut) {
		const int32_t* p3 = p2 + B + 1;
		const uint8_t* lv = (const uint8_t*)(o + L.oLev);
		for (size_t i = (size_t)p2[b] + lane; i < (size_t)p2[b + 1]; i += step) levelsOut[i] = lv[edge_slot(p2, p3, b, i, false)];
		for (size_t j = (size_t)p3[b] + lane; j < (size_t)p3[b + 1]; j += step) levelsOut[(size_t)E2 + j] = lv[edge_slot(p2, p3, b, j, true)];
	}
}

// one CTA per frame: q, t, then unpack_rounds.  statPer: stat slots per frame
__global__ void __launch_bounds__(BLOCK) k_unpack_poses(const PoseLayout L, int B, int R, int E2, int statPer, const double* in,
	double* qOut, double* tOut, uint8_t* levelsOut, int32_t* counts, cuba_iter_stat* stats, int32_t* nstats, const int32_t* status)
{
	if (*status) return;
	const int b = blockIdx.x, tid = threadIdx.x;
	const double* o = in + L.nIn;
	if (tid < 4) qOut[4 * (size_t)b + tid] = o[8 * (size_t)b + tid];
	else if (tid < 7) tOut[3 * (size_t)b + tid - 4] = o[8 * (size_t)b + tid];
	unpack_rounds(L, o, (const int32_t*)(in + L.oPtr), b, B, R, E2, statPer, tid, BLOCK, levelsOut, counts, stats, nstats);
}

// grid-stride over the problem records, the pair records and ptr
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
			in[k] = sim3_prob_rec(bt, k / s3::PROB, (int)(k % s3::PROB));
		} else {
			in[k] = sim3_pair_rec(bt, (k - nP) / s3::PAIR, (int)((k - nP) % s3::PAIR));
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

// one warp per point, and the pose table grid-stride
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
		in[L.oPose + k] = k < 8 * P ? pose_rec(bt.q, bt.t, p, c) : cam_rec(bt.cam, p, c);
	}
	if (b >= B) return;
	if (lane < 4) in[4 * (size_t)b + lane] = point_rec(bt, b, lane);
	const size_t i0 = (size_t)bt.ptr2[b], n2 = (size_t)bt.ptr2[b + 1] - i0, j0 = (size_t)bt.ptr3[b], n3 = (size_t)bt.ptr3[b + 1] - j0;
	const size_t m0 = edge_slot(bt.ptr2, bt.ptr3, b, i0, false), s0 = edge_slot(bt.ptr2, bt.ptr3, b, j0, true);
	for (size_t k = lane; k < 4 * n2; k += 32) in[L.oEdge + 4 * m0 + k] = point_mono_rec(bt, i0 + k / 4, (int)(k & 3));
	for (size_t k = lane; k < n2; k += 32) ip[m0 + k] = bt.iP2[i0 + k];
	for (size_t k = lane; k < 4 * n3; k += 32) in[L.oEdge + 4 * s0 + k] = point_stereo_rec(bt, j0 + k / 4, (int)(k & 3));
	for (size_t k = lane; k < n3; k += 32) ip[s0 + k] = bt.iP3[j0 + k];
}

// one warp per point: Xw, then unpack_rounds.  statPer: stat slots per point
__global__ void __launch_bounds__(BLOCK) k_unpack_points(const PointLayout L, int B, int R, int E2, int E3, int statPer, const double* in,
	double* XwOut, uint8_t* levelsOut, int32_t* counts, cuba_iter_stat* stats, int32_t* nstats, const int32_t* status)
{
	if (*status) return;
	const int b = blockIdx.x * POINTS_PER_BLOCK + (threadIdx.x >> 5), lane = threadIdx.x & 31;
	if (b >= B) return;
	const double* o = in + L.nIn;
	if (lane < 3) XwOut[3 * (size_t)b + lane] = o[4 * (size_t)b + lane];
	unpack_rounds(L, o, (const int32_t*)(in + L.oIdx) + (size_t)E2 + (size_t)E3, b, B, R, E2, statPer, lane, 32, levelsOut, counts, stats,
		nstats);
}

inline unsigned grid_for(size_t n) { return (unsigned)std::max<size_t>(1, std::min<size_t>(MAX_GRID, (n + BLOCK - 1) / BLOCK)); }

// ---- the host entry points' packers and unpackers: the same records, one problem after the other, in page-locked memory --------

inline void pack_poses(const cuba_pose_batch& bt, const PoseLayout& L, double* h)
{
	const size_t B = (size_t)bt.B;
	for (size_t b = 0; b < B; b++) {
		for (int c = 0; c < 8; c++) { h[8 * b + c] = pose_rec(bt.q, bt.t, b, c); h[L.oCam + 8 * b + c] = cam_rec(bt.cam, b, c); }
		for (size_t i = (size_t)bt.ptr2[b]; i < (size_t)bt.ptr2[b + 1]; i++) {
			double* d = h + L.oEdge + 8 * edge_slot(bt.ptr2, bt.ptr3, b, i, false);
			for (int c = 0; c < 8; c++) d[c] = pose_mono_rec(bt, i, c);
		}
		for (size_t j = (size_t)bt.ptr3[b]; j < (size_t)bt.ptr3[b + 1]; j++) {
			double* d = h + L.oEdge + 8 * edge_slot(bt.ptr2, bt.ptr3, b, j, true);
			for (int c = 0; c < 8; c++) d[c] = pose_stereo_rec(bt, j, c);
		}
	}
	int32_t* p = (int32_t*)(h + L.oPtr);
	memcpy(p, bt.ptr2, sizeof(int32_t) * (B + 1));
	memcpy(p + B + 1, bt.ptr3, sizeof(int32_t) * (B + 1));
}

inline void pack_sim3(const cuba_sim3_batch& bt, const Sim3Layout& L, double* h)
{
	for (size_t b = 0; b < (size_t)bt.B; b++)
		for (int c = 0; c < s3::PROB; c++) h[s3::PROB * b + c] = sim3_prob_rec(bt, b, c);
	for (size_t i = 0; i < (size_t)bt.N; i++)
		for (int c = 0; c < s3::PAIR; c++) h[L.oPair + s3::PAIR * i + c] = sim3_pair_rec(bt, i, c);
	memcpy(h + L.oPtr, bt.ptr, sizeof(int32_t) * ((size_t)bt.B + 1));
}

inline void pack_points(const cuba_point_batch& bt, const PointLayout& L, double* h)
{
	const size_t B = (size_t)bt.B, E = (size_t)bt.E2 + (size_t)bt.E3;
	for (size_t p = 0; p < (size_t)bt.P; p++)
		for (int c = 0; c < 8; c++) { h[L.oPose + 8 * p + c] = pose_rec(bt.q, bt.t, p, c); h[L.oCam + 8 * p + c] = cam_rec(bt.cam, p, c); }
	int32_t* hi = (int32_t*)(h + L.oIdx);
	for (size_t b = 0; b < B; b++) {
		for (int c = 0; c < 4; c++) h[4 * b + c] = point_rec(bt, b, c);
		for (size_t i = (size_t)bt.ptr2[b]; i < (size_t)bt.ptr2[b + 1]; i++) {
			const size_t k = edge_slot(bt.ptr2, bt.ptr3, b, i, false);
			for (int c = 0; c < 4; c++) h[L.oEdge + 4 * k + c] = point_mono_rec(bt, i, c);
			hi[k] = bt.iP2[i];
		}
		for (size_t j = (size_t)bt.ptr3[b]; j < (size_t)bt.ptr3[b + 1]; j++) {
			const size_t k = edge_slot(bt.ptr2, bt.ptr3, b, j, true);
			for (int c = 0; c < 4; c++) h[L.oEdge + 4 * k + c] = point_stereo_rec(bt, j, c);
			hi[k] = bt.iP3[j];
		}
	}
	memcpy(hi + E, bt.ptr2, sizeof(int32_t) * (B + 1));
	memcpy(hi + E + B + 1, bt.ptr3, sizeof(int32_t) * (B + 1));
}

// ---- one launch of each LM kernel on packed records: `in` is the layout's input area, `out` its results (the host entry points'
// device buffers, the device entry points' workspace).  stats: whether the caller wants stats.

inline void launch_poses(const PoseLayout& L, int B, const pb::Schedule& s, const double* in, double* out, bool stats, cudaStream_t st)
{
	pb::Args a;
	a.B = B;
	a.pose = in; a.cam = in + L.oCam; a.edge = in + L.oEdge;
	a.ptr2 = (const int*)(in + L.oPtr); a.ptr3 = a.ptr2 + (size_t)B + 1;
	a.poseOut = out;
	a.stats = stats ? (lm::IterStat*)(out + L.oStat) : nullptr;
	a.counts = (int*)(out + L.oInt); a.nstats = a.counts + 4 * (size_t)B * (size_t)s.n;
	a.level = (unsigned char*)(out + L.oLev);
	pb::k_pose_batch<<<(unsigned)B, lm::BLOCK, 0, st>>>(a, s);
}

inline void launch_sim3(const Sim3Layout& L, int B, const s3::Params& p, const double* in, double* out, bool stats, cudaStream_t st)
{
	s3::Args a;
	a.B = B;
	a.prob = in; a.pair = in + L.oPair; a.ptr = (const int*)(in + L.oPtr);
	a.Sout = out;
	a.stats = stats ? (lm::IterStat*)(out + L.oStat) : nullptr;
	a.ninliers = (int*)(out + L.oInt); a.nstats = a.ninliers + B;
	a.level = (unsigned char*)(out + L.oLev);
	s3::k_sim3_batch<<<(unsigned)B, lm::BLOCK, 0, st>>>(a, p);
}

inline void launch_points(const PointLayout& L, int B, size_t E, const pb::Schedule& s, const double* in, double* out, bool stats,
	cudaStream_t st)
{
	ptb::Args a;
	a.B = B;
	a.Xw = in; a.pose = in + L.oPose; a.cam = in + L.oCam; a.edge = in + L.oEdge;
	a.iP = (const int*)(in + L.oIdx); a.ptr2 = a.iP + E; a.ptr3 = a.ptr2 + (size_t)B + 1;
	a.XwOut = out;
	a.stats = stats ? (lm::IterStat*)(out + L.oStat) : nullptr;
	a.counts = (int*)(out + L.oInt); a.nstats = a.counts + 4 * (size_t)B * (size_t)s.n;
	a.level = (unsigned char*)(out + L.oLev);
	ptb::k_point_batch<<<(unsigned)(((size_t)B + ptb::WARPS - 1) / ptb::WARPS), lm::BLOCK, 0, st>>>(a, s);
}

}  // namespace bio
}  // namespace cuba_b200
