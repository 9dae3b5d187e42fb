// cuba_landmark_refine.cuh -- structure-only refinement of the engine's own landmarks in place (Engine::optimize_landmarks).
//
// k_refine_landmarks runs k_point_batch's per-point problem (ptb::Point, ptb::run_schedule) on the free landmarks of the problem the
// engine holds: one WARP per listed landmark l, over l's run [lmPtr[l], lmPtr[l+1]) of the landmark-major edge stream, against the
// poses of pose[cur] / cam held fixed.  Nothing is packed: per edge the warp reads the measurement (e_mx / e_my / e_mz), the caller's
// omega (e_om0, never the masked e_om), the pose and the stereo bit (e_ip), and the level byte lvLevel[e_user[k]], which the outlier
// test rewrites in place.  The committed position goes to Xw[cur].
//
// Counts: per CTA and round, the four counts of its warps summed in a fixed order (integers, no atomics), [round][CTA][4], which
// lv::k_sum_counts reduces round by round.  A landmark outside the rank's shard [lmBeg, lmEnd) is not refined; its per-landmark
// outputs are written as 0.
//
// The device entry's list is checked by k_check_landmarks first: an entry outside [0, numL) or repeated (an integer atomic on a
// per-landmark mark) sets the status word, and k_refine_landmarks then writes nothing -- two warps on one landmark would race.
#pragma once

#include "cuba_point_batch.cuh"

namespace cuba_b200 {
namespace ptb {

constexpr int BAD_INDEX = 1;      // status bits of k_check_landmarks: an entry outside [0, numL)
constexpr int REPEATED = 2;       // an entry listed twice

// The edges of landmark l in the engine's landmark-major stream: e0 = lmPtr[l] .. lmPtr[l+1], in the stream's order (ascending pose,
// then edge id); levels in edge-id order
struct StreamEdges {
	const double* mx;
	const double* my;
	const double* mz;
	const double* om;                 // e_om0: the caller's omega
	const int* ip;                    // pose | 0x80000000 for a stereo edge
	const int* user;                  // edge id
	unsigned char* level;             // [E], edge-id order
	int e0;

	__device__ __forceinline__ int pose(int k, bool& stereo) const
	{
		const int ipf = ip[e0 + k];
		stereo = ipf < 0;
		return ipf & 0x7fffffff;
	}
	__device__ __forceinline__ void meas(int k, bool stereo, double m[3], double& om_) const
	{
		m[0] = mx[e0 + k]; m[1] = my[e0 + k]; m[2] = stereo ? mz[e0 + k] : 0.0;
		om_ = om[e0 + k];
	}
	__device__ __forceinline__ unsigned char* slot(int k) const { return level + user[e0 + k]; }
};

struct LandmarkArgs {
	int n;                            // list entries
	const int* list;                  // [n] landmark of entry b; null: entry b is landmark b
	int lmBeg, lmEnd;                 // the rank's shard
	const double* pose;               // pose[cur], cam: [Pall][8]
	const double* cam;
	double* Xw;                       // Xw[cur]: [Lall][4]
	const double* mx;
	const double* my;
	const double* mz;
	const double* om0;
	const int* ip;
	const int* user;
	const int* lmPtr;                 // [Lall+1], the rank's local stream
	unsigned char* level;             // lvLevel
	const int* status;                // non-zero: a bad list, nothing is written; null on the host entry (checked there)
	int* partial;                     // [s.n][gridDim.x][4]
	int* nstats;                      // [n][s.n] or null
	lm::IterStat* stats;              // [n][s.statOff[s.n]] or null
};

__global__ void __launch_bounds__(lm::BLOCK) k_refine_landmarks(const LandmarkArgs a, const pb::Schedule s)
{
	__shared__ int s_cnt[WARPS][pb::MAX_ROUNDS][4];
	if (a.status && *a.status) return;    // the same word for every thread: no barrier is skipped by part of a CTA
	const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int b = blockIdx.x * WARPS + w;
	const int l = b < a.n ? (a.list ? a.list[b] : b) : -1;
	const int S = s.statOff[s.n];
	if (l >= a.lmBeg && l < a.lmEnd) {
		const int e0 = a.lmPtr[l], n = a.lmPtr[l + 1] - e0;
		const StreamEdges ed = { a.mx, a.my, a.mz, a.om0, a.ip, a.user, a.level, e0 };
		double Xin[3], X[3];
#pragma unroll
		for (int i = 0; i < 3; i++) X[i] = Xin[i] = a.Xw[4 * (size_t)l + i];
		int included = 0;
		for (int k = lane; k < n; k += 32) included += *ed.slot(k) == 0;
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) included += __shfl_xor_sync(0xffffffffu, included, o);
		run_schedule(a.pose, a.cam, ed, n, s, Xin, X, included, a.stats ? a.stats + (size_t)b * S : nullptr,
			[&](int rd, int nIt, const int c4[4]) {
				if (lane < 4) s_cnt[w][rd][lane] = lane == 0 ? c4[0] : lane == 1 ? c4[1] : lane == 2 ? c4[2] : c4[3];
				if (lane == 0 && a.nstats) a.nstats[(size_t)b * s.n + rd] = nIt;
			});
		if (lane < 3) a.Xw[4 * (size_t)l + lane] = lane == 0 ? X[0] : lane == 1 ? X[1] : X[2];
	} else {
		for (int i = lane; i < 4 * s.n; i += 32) s_cnt[w][i >> 2][i & 3] = 0;
		if (b < a.n) {      // another rank's landmark: zero outputs
			for (int i = lane; i < s.n; i += 32)
				if (a.nstats) a.nstats[(size_t)b * s.n + i] = 0;
			if (a.stats)
				for (int i = lane; i < S; i += 32) a.stats[(size_t)b * S + i] = lm::IterStat{ 0, 0, 0.0, 0.0, 0, 0 };
		}
	}
	__syncthreads();
	if (threadIdx.x < 4 * s.n) {
		const int rd = threadIdx.x >> 2, k = threadIdx.x & 3;
		int v = 0;
#pragma unroll
		for (int i = 0; i < WARPS; i++) v += s_cnt[i][rd][k];
		a.partial[((size_t)rd * gridDim.x + blockIdx.x) * 4 + k] = v;
	}
}

// the device entry's list: an entry outside [0, numL) or repeated sets its bit in *status (mark: [numL] zeros on entry)
__global__ void k_check_landmarks(const int* __restrict__ list, int n, int numL, int* mark, int* status)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const int l = list[i];
	if (l < 0 || l >= numL) { atomicOr(status, BAD_INDEX); return; }
	if (atomicAdd(mark + l, 1) != 0) atomicOr(status, REPEATED);
}

}  // namespace ptb
}  // namespace cuba_b200
