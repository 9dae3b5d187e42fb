// cuba_engine.cu -- the engine behind the C ABI of include/cuba_b200.h: device memory, the host LM
// control loop (reference src/cuda_bundle_adjustment.cpp:793-857) and the kernel launches.
//
// No CPU fallback: every compute entry point needs a CUDA device and fails loudly without one.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/cuba_b200.h"
#include "cuba_kernels.cuh"
#include "cuba_pcg2.cuh"
#include "cuba_pcg3.cuh"
#include "cuba_pcg4.cuh"
#include "cuba_pcg5.cuh"
#include "cuba_pcg5t.cuh"
#include "cuba_coarse.cuh"
#include "cuba_dense_chol.cuh"
#include "cuba_peer_reduce.cuh"
#include "cuba_jh4.cuh"
#include "cuba_levels.cuh"
#include "cuba_pose_batch.cuh"
#include "cuba_sim3_batch.cuh"
#include "cuba_point_batch.cuh"
#include "cuba_landmark_refine.cuh"
#include "cuba_batch_io.cuh"
#include "cuba_problem_io.cuh"
#include "cuba_schur3.cuh"
#include "cuba_schur5.cuh"
#include "cuba_structure.h"
#include "cuba_structure_gpu.cuh"

namespace cuba_b200 {

static thread_local std::string g_err;
static int fail(int code, const std::string& msg) { g_err = msg; return code; }
// the direct solver holds the whole reduced camera system in fp64 tiles: at most dchol::MAX_POSES free poses
static int dense_cap_error(int numP)
{
	return fail(CUBA_ERR_INVALID, "set_problem: the dense Cholesky solver takes at most " + std::to_string(dchol::MAX_POSES) + " free poses, this problem has numP = "
		+ std::to_string(numP) + " (choose CUBA_SOLVER_PCG)");
}

// fixed shared-memory footprint of k_pcg3 (a superset of k_pcg2's): r,s per needed column, p,y per own row, index lists
static size_t pcg3_fixed_bytes(int needMax, int maxRows, size_t scalar)
{
	return (size_t)needMax * (12 * scalar + 8) + (size_t)maxRows * (12 * scalar + 4) + ((size_t)maxRows + 1) * 4 + (size_t)PCG3_CHUNK * 6 * scalar;
}

// columns of w a k_pcg5 / k_pcg5t layout's staging region `cc` holds between passes (it ends where the next region, rc, begins)
template <typename L>
static int32_t w_staging_columns(const L& lay) { return (int32_t)((lay.rc - lay.cc) / (6 * sizeof(double))); }

// The dimensions of a k_pcg5 plan over W ranks that do not depend on the launch shape (capBlocks and zhInSmem stay 0).
static Pcg5Dims pcg5_plan_dims(const Pcg5Plan& plan, int W)
{
	const int G = plan.G, nc = 6 * plan.A, NR = 3 + 6 * (G / plan.gs);
	Pcg5Dims d{};
	d.needMax = plan.P.needMax; d.maxRows = plan.P.maxRows; d.nc = nc; d.maxNeedAgg = plan.C.maxNeedAgg;
	d.npv = std::max(std::max(G * p5t::pcg5t_np(plan.apc), W * NR), 6 * plan.C.maxNeedAgg); d.nls = NR;
	d.sliceRows = (nc + G - 1) / G;
	return d;
}

// Pcg5Dims of the tuned one-GPU shape (cuba_pcg5t.cuh) for a plan on one GPU; p5t::pcg5t_fit sizes the caches
static p5t::Pcg5Dims pcg5t_plan_dims(const Pcg5Plan& plan)
{
	const Pcg5Dims d = pcg5_plan_dims(plan, 1);
	p5t::Pcg5Dims t{};
	t.needMax = d.needMax; t.maxRows = d.maxRows; t.nc = d.nc; t.maxNeedAgg = d.maxNeedAgg;
	t.npv = d.npv; t.nls = d.nls; t.sliceRows = d.sliceRows;
	t.ccCap = p5t::pcg5t_cc_cap(plan.P.blkMax);
	t.sqWords = p5t::pcg5t_np(plan.apc) * (p5t::Pcg5Shape::BLOCK / 32);
	return t;
}

// the block-Jacobi dimensions of a k_pcg5 / k_pcg5t shape from its two-level ones: no coarse level, three words per rank summary
template <typename D>
static D block_jacobi_dims(D d, int G, int W)
{
	d.nc = 0; d.maxNeedAgg = 0; d.zhInSmem = 0; d.sliceRows = 0; d.nls = 3; d.npv = std::max(G * 3, W * 3);
	return d;
}

// the kernel that inverts a coarse matrix of A aggregates: one CTA while the packed triangle fits its shared memory, the blocked
// sweep on the whole chip above
static int coarse_kernel(int A) { return A > PCG4_MAXAGG1 ? CUBA_COARSE_KERNEL_DENSE : CUBA_COARSE_KERNEL_INVERT; }

// The J+H and Schur kernels of an engine (stage_choice)
struct StageChoice {
	bool jh4 = false;                        // the warp-tile pass k_linearize_landmark4 (cuba_jh4.cuh), fp64 only
	int jh4Stages = 2, jh4MinB = 4;          // its pipeline stages and CTAs per SM (the grid's, also under mixed precision)
	int tileSize = LM_TILE, minBlocks = 4;   // first-generation landmark tiles: edges, CTAs per SM (k_backsub runs on them too)
	bool mixed = false;                      // Hpl in fp32: k_linearize_landmark4<4, 2, 0, true> whatever the shape
	bool schur5 = false;                     // the tensor-pipe Schur is asked for and the engine can run it (alloc_system: useSchur5)
};
// The only reader of cfg.reserved[2] (J+H kernel), reserved[3] (Schur kernel) and use_fp32 == 2; refuses a value that names no kernel.
// reserved[2]: 0 = k_linearize_landmark4, two stages, 4 CTAs of 4 warps per SM; 7 = three stages; 8 / 9 = 5 / 6 CTAs per SM; 1..4 = the
// first generation (tileOf x minBOf).  The fp32 engine's default is 128 x 6 first-generation tiles: the warp tiles' bulk copy needs
// 16-byte multiples, which 144-byte fp64 blocks are and 72-byte fp32 blocks are not.  reserved[3] = 5, the tensor-pipe Schur
// (cuba_schur5.cuh), is opt-in: 12 % faster than k_schur3 on the banded 5 M-edge graph, on par on kitti00_shaped, 2x slower on the real
// ba_kitti_00 whose loop closures leave 4.4 products per (tile, destination) segment.
static int stage_choice(const cuba_config& c, bool fp64, StageChoice& s)
{
	const int r2 = c.reserved[2], r3 = c.reserved[3];
	if (r2 < 0 || r2 == 5 || r2 == 6 || r2 > 9)
		return fail(CUBA_ERR_INVALID, "create: reserved[2] = " + std::to_string(r2) + " names no J+H kernel (0..4, 7..9)");
	if (r3 != 0 && r3 != 3 && r3 != 5)
		return fail(CUBA_ERR_INVALID, "create: reserved[3] = " + std::to_string(r3) + " names no Schur kernel (0, 3, 5)");
	static const int tileOf[10] = { LM_TILE, 256, 256, 128, 128, 0, 0, LM_TILE, LM_TILE, LM_TILE }, minBOf[10] = { 4, 2, 3, 4, 6, 0, 0, 4, 4, 4 };
	s.jh4 = (r2 == 0 || r2 >= 7) && fp64;
	s.jh4Stages = r2 == 7 ? 3 : 2;
	s.jh4MinB = r2 == 8 ? 5 : (r2 == 9 ? 6 : 4);
	s.tileSize = r2 == 0 && !fp64 ? 128 : tileOf[r2];
	s.minBlocks = r2 == 0 && !fp64 ? 6 : minBOf[r2];
	s.mixed = c.use_fp32 == 2 && s.jh4;
	s.schur5 = r3 == 5 && c.reserved[1] != 1 && c.use_fp32 != 2 && fp64;
	return CUBA_OK;
}

#define CUDA_TRY(expr)                                                                                      \
	do {                                                                                                    \
		cudaError_t _e = (expr);                                                                            \
		if (_e != cudaSuccess) {                                                                            \
			char _b[512];                                                                                   \
			snprintf(_b, sizeof(_b), "%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
			return fail(CUBA_ERR_CUDA, _b);                                                                 \
		}                                                                                                   \
	} while (0)

// launches a 1-D kernel over n items on the engine's stream (used inside Engine<T> member functions)
#define KLAUNCH(kernel, n, ...)                                                             \
	do {                                                                                     \
		if ((n) > 0) {                                                                       \
			kernel<<<sgpu::grid_for(n), sgpu::BLK, 0, stream>>>(__VA_ARGS__);                 \
			launches++;                                                                      \
			CUDA_TRY(cudaGetLastError());                                                    \
		}                                                                                    \
	} while (0)

static thread_local long long g_h2dBytes = 0, g_d2hBytes = 0;   // host<->device traffic of this thread's engines

// Pinned staging arena for the many small host->device uploads of the PCG setup: a cudaMemcpyAsync from pageable
// memory is staged (and effectively synchronous) inside the driver; from the arena it is a plain DMA.
struct PinnedArena {
	char* p = nullptr; size_t cap = 0, off = 0;
	~PinnedArena() { if (p) cudaFreeHost(p); }
	void reset() { off = 0; }
	// returns nullptr when the arena would have to grow while earlier copies may still read it: the caller falls back
	void* put(const void* src, size_t bytes)
	{
		const size_t o = (off + 255) & ~(size_t)255;
		if (o + bytes > cap) {
			if (off != 0) return nullptr;
			if (p) cudaFreeHost(p);
			cap = std::max<size_t>(2 * (o + bytes), (size_t)1 << 20);
			if (cudaMallocHost((void**)&p, cap) != cudaSuccess) { p = nullptr; cap = 0; return nullptr; }
		}
		memcpy(p + o, src, bytes);
		off = o + bytes;
		return p + o;
	}
};

// grow-only page-locked host buffer (the staging area of one packed copy)
struct PinnedBuf {
	char* p = nullptr; size_t cap = 0;
	PinnedBuf() {}
	PinnedBuf(const PinnedBuf&) = delete;
	PinnedBuf& operator=(const PinnedBuf&) = delete;
	~PinnedBuf() { if (p) cudaFreeHost(p); }
	cudaError_t grow(size_t bytes)
	{
		if (p && bytes <= cap) return cudaSuccess;
		if (p) cudaFreeHost(p);
		p = nullptr; cap = 0;
		const cudaError_t e = cudaMallocHost((void**)&p, std::max<size_t>(bytes, 256));
		if (e == cudaSuccess) cap = std::max<size_t>(bytes, 256);
		else p = nullptr;
		return e;
	}
};

template <typename U>
struct DBuf {
	U* p = nullptr; size_t n = 0, cap = 0;
	bool view = false;   // a window into another DBuf's allocation (fused collectives): never freed, never grown here
	DBuf() {}
	DBuf(const DBuf&) = delete;
	DBuf& operator=(const DBuf&) = delete;
	~DBuf() { release(); }
	void release() { if (p && !view) cudaFree(p); p = nullptr; n = 0; cap = 0; view = false; }
	void alias(U* q, size_t count) { release(); p = q; n = count; cap = count; view = true; }
	// grow-only: re-initialising an engine with a problem of the same (or smaller) size allocates nothing
	cudaError_t alloc(size_t count)
	{
		if (p && count <= cap && !view) { n = count; return cudaSuccess; }
		release();
		n = count; cap = count ? count : 1;
		return cudaMalloc((void**)&p, sizeof(U) * cap);
	}
	cudaError_t upload(const U* h, size_t count, cudaStream_t s)
	{
		cudaError_t e = alloc(count);
		if (e != cudaSuccess || !count) return e;
		g_h2dBytes += (long long)(sizeof(U) * count);
		return cudaMemcpyAsync(p, h, sizeof(U) * count, cudaMemcpyHostToDevice, s);
	}
	cudaError_t upload(const std::vector<U>& h, cudaStream_t s) { return upload(h.data(), h.size(), s); }
	// from a caller's device array on the same device: no host traffic, nothing counted
	cudaError_t copy(const U* d, size_t count, cudaStream_t s)
	{
		cudaError_t e = alloc(count);
		if (e != cudaSuccess || !count) return e;
		return cudaMemcpyAsync(p, d, sizeof(U) * count, cudaMemcpyDeviceToDevice, s);
	}
	// through the pinned arena when one is given
	cudaError_t upload(const std::vector<U>& h, cudaStream_t s, PinnedArena* arena)
	{
		const void* src = h.empty() || !arena ? nullptr : arena->put(h.data(), sizeof(U) * h.size());
		return upload(src ? (const U*)src : h.data(), h.size(), s);
	}
	operator U*() const { return p; }
};

// One coarse level of a two-level PCG (cuba_coarse.cuh): the device lists of a CoarsePartition, the packed coarse matrix Ac
// (fp64) and its inverse (fp32), and when that inverse was built.  k_pcg4 and k_pcg5 each own one.
struct CoarseLevel {
	int A = 0;
	DBuf<int> aggRow, naPtr, naList, needAgg, rowOf, cbPtr, cbList;
	DBuf<double> AcP;
	DBuf<float> AcInv;
	bool valid = false;   // AcInv holds the inverse coarse matrix of an earlier solve of this problem
	int age = 0;          // two-level solves since the coarse matrix was last rebuilt
	double lambda = 0;    // damping of that rebuild
	long long rebuilds = 0;  // since set_problem (k_pcg5's rebuild log in cInfo)
	void forget() { valid = false; age = 0; }
	// the lists of CP (build_coarse_lists run), Ac and Ac^-1 sized for its A; no inverse yet
	int upload(const CoarsePartition& CP, cudaStream_t s, PinnedArena* arena)
	{
		A = CP.A;
		forget();
		CUDA_TRY(aggRow.upload(CP.aggRow, s, arena)); CUDA_TRY(naPtr.upload(CP.naPtr, s, arena)); CUDA_TRY(naList.upload(CP.naList, s, arena));
		CUDA_TRY(needAgg.upload(CP.needAgg, s, arena)); CUDA_TRY(rowOf.upload(CP.rowOf, s, arena));
		CUDA_TRY(cbPtr.upload(CP.cbPtr, s, arena)); CUDA_TRY(cbList.upload(CP.cbList, s, arena));
		CUDA_TRY(AcP.alloc((size_t)A * (A + 1) / 2 * 36)); CUDA_TRY(AcInv.alloc(36 * (size_t)A * A));
		return CUBA_OK;
	}
};

// cudaIpc mappings of one device allocation of every rank (ipcExchange); the own entry is the local allocation
struct PeerMap {
	void* base[PCG5_MAXWORLD] = { nullptr };
	void* mappedFor = nullptr;   // local allocation the mappings were exchanged for
	void close(int rank)
	{
		for (int r = 0; r < PCG5_MAXWORLD; r++) { if (base[r] && r != rank) cudaIpcCloseMemHandle(base[r]); base[r] = nullptr; }
		mappedFor = nullptr;
	}
};

// ---- NCCL through dlopen: single-GPU users never need the library ---------------------------------
struct Nccl {
	void* lib = nullptr;
	typedef struct { char internal[128]; } UniqueId;
	int (*GetUniqueId)(UniqueId*) = nullptr;
	int (*CommInitRank)(void**, int, UniqueId, int) = nullptr;
	int (*CommDestroy)(void*) = nullptr;
	int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
	int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
	int (*Broadcast)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
	int (*GroupStart)() = nullptr;
	int (*GroupEnd)() = nullptr;
	const char* (*GetErrorString)(int) = nullptr;
	bool load(std::string& why)
	{
		if (lib) return true;
		const char* names[] = { "libnccl.so.2", "libnccl.so" };
		for (const char* nme : names) { lib = dlopen(nme, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
		if (!lib) { why = std::string("dlopen libnccl.so.2 failed: ") + dlerror(); return false; }
		GetUniqueId = (int (*)(UniqueId*))dlsym(lib, "ncclGetUniqueId");
		CommInitRank = (int (*)(void**, int, UniqueId, int))dlsym(lib, "ncclCommInitRank");
		CommDestroy = (int (*)(void*))dlsym(lib, "ncclCommDestroy");
		AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(lib, "ncclAllReduce");
		AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(lib, "ncclAllGather");
		Broadcast = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(lib, "ncclBroadcast");
		GroupStart = (int (*)())dlsym(lib, "ncclGroupStart");
		GroupEnd = (int (*)())dlsym(lib, "ncclGroupEnd");
		GetErrorString = (const char* (*)(int))dlsym(lib, "ncclGetErrorString");
		if (!GetUniqueId || !CommInitRank || !CommDestroy || !AllReduce || !AllGather || !Broadcast || !GroupStart || !GroupEnd) { why = "libnccl lacks expected symbols"; return false; }
		return true;
	}
};
static Nccl g_nccl;
enum { NCCL_INT8 = 0, NCCL_FLOAT32 = 7, NCCL_FLOAT64 = 8, NCCL_SUM = 0, NCCL_MAX = 2 };

struct Scalars { double v[8]; unsigned long long maxdiag; PcgStatus pcg; };

// Every C ABI entry point runs on the engine's own device, whatever the calling thread's current device is
// (two engines on two GPUs in one thread; a host that calls torch.cuda.set_device between calls).
struct DevGuard {
	int prev = -1, dev;
	explicit DevGuard(int d) : dev(d) { if (cudaGetDevice(&prev) != cudaSuccess) prev = -1; if (prev != dev) cudaSetDevice(dev); }
	~DevGuard() { if (prev >= 0 && prev != dev) cudaSetDevice(prev); }
};

struct EngineBase {
	virtual ~EngineBase() {}
	cuba_config cfg{};
	int rk_type[2] = { 0, 0 };
	double rk_delta[2] = { 0, 0 };
	int rank = 0, world = 1;
	bool structureReuse = true;   // cuba_engine_set_structure_reuse
	int linSolver = CUBA_SOLVER_PCG;   // cuba_engine_set_linear_solver: applies from the next set_problem
	long long structureReuses = 0;
	int devOrdinal = 0;      // CUDA device every call of this engine runs on (set once in init)
	void* comm = nullptr;
	bool haveProblem = false;
	cudaStream_t stream = nullptr;   // the engine's own (init)
	long long launches = 0;
	double prof[CUBA_PROF_NUM] = { 0 };
	// the batched LM kernels' packed batch and packed results, device and page-locked host copies, grown to the largest call; the
	// host entry of optimize_landmarks moves its list and per-landmark outputs through them too
	DBuf<double> batchIn, batchOut;
	PinnedBuf batchHostIn, batchHostOut;

	virtual int set_problem(const cuba_problem* p) = 0;
	virtual int set_state(const double* q, const double* t, const double* Xw) = 0;
	virtual int get_sizes(cuba_sizes* out) const = 0;
	virtual int reset_state() = 0;
	virtual int flush_l2() = 0;
	virtual int optimize(int niter, cuba_iter_stat* stats, int* nstats) = 0;
	virtual int get_state(double* q, double* t, double* Xw) = 0;
	virtual int get_chi2(double* out) = 0;
	virtual int get_profile(double* sec) = 0;
	virtual int stage_linearize(double* chi) = 0;
	virtual int stage_max_diagonal(double* md) = 0;
	virtual int stage_solve(double lambda, int* iters, int* ok) = 0;
	virtual int stage_update(double lambda, double* chi, double* scale) = 0;
	virtual int stage_commit(int accept) = 0;
	virtual int stage_chi2(double* chi) = 0;
	virtual int dbg_hpl_structure(int32_t* colPtr, int32_t* rowInd, int32_t* e2h) = 0;
	virtual int dbg_hsc_structure(int32_t* rowPtr, int32_t* colInd) = 0;
	virtual int dbg_system(double* Hpp, double* bp, double* Hll, double* bl, double* Hpl) = 0;
	virtual int dbg_schur(double* Hsc, double* bsc, double* invHll) = 0;
	virtual int dbg_delta(double* xp, double* xl) = 0;
	virtual int bench_stage(int stage, int reps, int flush, double lambda, double* ms) = 0;
	virtual int dbg_pcg_timing(long long* out, int maxCtas) = 0;
	virtual int dbg_pcg_info(int32_t* info, double* coarseLambda) = 0;
	virtual int dbg_coarse(int32_t* rowAgg, double* AcP, float* AcInv) = 0;
	virtual int dbg_coarse_inverse(const double* AcP, int A, float* AcInv, int* info) = 0;
	virtual int dbg_dense_solve(const double* S, const double* b, int n, double* x, int* info) = 0;
	virtual int dbg_peer_allreduce(int world, size_t n, int calls, const double* parts, double* out) = 0;
	virtual int dbg_pcg5_ranks(int world, int twoLevel, int nsolves, double* x, int32_t* status, int32_t* plan, int32_t* aggRow, float* AcInv) = 0;
	virtual int set_edge_levels(const uint8_t* levels) = 0;
	virtual int get_edge_levels(uint8_t* levels) = 0;
	virtual int classify_edges(double chi2Mono, double chi2Stereo, int flags, int32_t* counts) = 0;
	// the problem on device-resident arrays, ordered after `caller`'s work (NULL: the engine's stream)
	virtual int set_problem_device(const cuba_problem* p, cudaStream_t caller) = 0;
	virtual int set_state_device(const double* q, const double* t, const double* Xw, cudaStream_t caller) = 0;
	virtual int get_state_device(double* q, double* t, double* Xw, cudaStream_t caller) = 0;
	virtual int get_chi2_device(double* out, cudaStream_t caller) = 0;
	virtual int set_edge_levels_device(const uint8_t* levels, cudaStream_t caller) = 0;
	virtual int get_edge_levels_device(uint8_t* levels, cudaStream_t caller) = 0;
	// the batched LM kernels on host arrays (cuba_batch_io.cuh): always fp64, on the stream; they touch nothing of the engine's
	// problem.  The batch was validated by the caller and has B > 0.
	int optimize_poses(const cuba_pose_batch& bt, const pb::Schedule& s, double* qOut, double* tOut, uint8_t* levelsOut, int32_t* counts,
		cuba_iter_stat* stats, int32_t* nstats);
	int optimize_sim3(const cuba_sim3_batch& bt, const s3::Params& p, double* qOut, double* tOut, double* sOut, uint8_t* levelsOut,
		int32_t* ninliers, cuba_iter_stat* stats, int32_t* nstats);
	int optimize_points(const cuba_point_batch& bt, const pb::Schedule& s, double* XwOut, uint8_t* levelsOut, int32_t* counts,
		cuba_iter_stat* stats, int32_t* nstats);
	int batch_grow(size_t nIn, size_t nOut);
	int batch_up(size_t nIn);
	int batch_down(size_t nOut);
	// structure-only refinement of the held problem's free landmarks in place; dev: list, stats and nstats are device pointers
	virtual int optimize_landmarks(const int32_t* list, int n, const pb::Schedule& s, int32_t* counts, cuba_iter_stat* stats,
		int32_t* nstats, bool dev, cudaStream_t caller) = 0;
	virtual int num_free_landmarks() const = 0;
	virtual bool fp32() const = 0;
};

template <typename T>
struct Engine : EngineBase {
	Structure S;
	int numSMs = 0;
	int smemMax = 0;        // opt-in dynamic shared memory of one CTA
	int ntiles = 0, nPoseBlocks = 0, nChiBlocks = 0;
	StageChoice stages;     // of cfg (init)
	// The warp-tile J+H pass of a structure (setup_jh4, setup_jh4_finish), and its kernel of the choice (init sets the attribute once)
	struct Jh4Run {
		int ntiles = 0, grid = 0; const void* fn = nullptr; size_t smem = 0;
		int* host = nullptr;         // pinned: {number of warp tiles, any cut landmark}
		bool pending = false;        // setup_jh4 queued the read-back of `host`
		DBuf<int> levels, start, pieces, base, tilePose, tilePieces, pieceCount, flag;
		DBuf<jh4::WTile> tile; DBuf<jh4::Rec> rec; DBuf<double> bigPartial;
	};
	Jh4Run wt;
	// The landmark-tile Schur complement on the tensor pipe of a structure (setup_schur5)
	struct Schur5Run {
		int ntiles = 0;
		DBuf<TileInfo> tileInfo; DBuf<int4> segRec; DBuf<unsigned int> off;
		DBuf<unsigned long long> key, keyS, key3, key3S;
		DBuf<int> tileLm, val, valS, head, segId, segStart, segTile, segDest, val3, val3S, segRank, rankDest, tileSegPtr, destSegPtr, p2i, p2j;
		DBuf<schur5::Counts> counts;
		DBuf<T> partial;
	};
	Schur5Run s5;
	bool useSchur5 = false;   // this structure's Schur runs on the tensor pipe; k_schur3 (cuba_schur3.cuh) otherwise
	int cur = 0;            // current state buffer
	bool trialValid = false;
	// state
	DBuf<T> pose[2], Xw[2], cam, pose0, Xw0;
	// edge streams
	DBuf<T> e_mx, e_my, e_mz, e_om, p_mx, p_my, p_mz, p_om;
	DBuf<int> tilePtr;   // run pointers seen by the landmark tiles (see k_tile_ptr)
	DBuf<int> e_ip, e_il, e_hpl, e_user, lmPtr, tileLm, hplLm, posePtr, p_il;
	// system
	DBuf<T> Hpp, bp, Hll, bl, Hpl, invHll, fVal, bsc, xp, xl;
	DBuf<T> uVal;            // landmark-sharded runs: upper Hsc blocks | bsc, the buffer of the per-trial all-reduce
	DBuf<float> HplF;        // mixed precision (stages.mixed): the Hpl blocks in fp32, 20 floats per block
	bool upperReduce = false;   // k_schur3 writes the upper blocks into uVal; one all-reduce of uVal | bsc, then k_expand_upper
	DBuf<int> prodPtr, prodI, prodJ, prodL, blkRow, blkCol, u2f, u2fT, fRowPtr, fColInd;
	// One block-Jacobi solve set up on the device (setup_pcg3): the row partition's lists, L^-1, the eight vectors, the partial board
	// and k_pcg3's flags, and the launch shape of k_pcg3 / k_pcg2 (cuba_pcg3.cuh, cuba_pcg2.cuh), the solve every other one falls back to
	struct Pcg3Run {
		int G = 0, cap = 0, needMax = 0, maxRows = 0; size_t smem = 0;   // cap: blocks of A^ cached in shared memory
		bool pcg3 = false;                               // k_pcg3 fits (one (row, component) pair per thread); k_pcg2 otherwise
		DBuf<int> ctaRow, needPtr, needCol, local;
		DBuf<T> Linv, R0, R1, S0, S1, W0, W1, P, Y;
		DBuf<double> partial;
		DBuf<unsigned long long> flags;                  // k_pcg3: [wFlag 2*6numP*2 | pFlag 2*2G*2 | abort word]
	};
	// One k_pcg4 solve set up on the device (setup_pcg4): its coarse level, Z^, partial board and shape; the rest is p3's
	struct Pcg4Run {
		bool ok = false; int gs = 1, maxNeedAgg = 0, cap = 0, sliceInSmem = 0, zhInSmem = 0; size_t smem = 0;
		CoarseLevel coarse;
		DBuf<T> Zhat; DBuf<double> part;
	};
	Pcg3Run p3;
	Pcg4Run p4;
	// Scratch the PCG solves share, each DBuf grown to the largest size asked for: A^ (setup_pcg3, setup_pcg5); the coarse basis Zx,
	// U [36 nfull] and k_coarse_dense's tiles of a coarse rebuild (setup_pcg4, setup_pcg5); the rebuild flags, slot 0 k_pcg4's, slots
	// 1..P5_INFO_LOG k_pcg5's log (setup_pcg4: one slot; setup_pcg5: all, zeroed); -DCUBA_PCG_TIMING's per-CTA counters (each launch)
	DBuf<T> fHat, cZx;
	DBuf<double> cU, cdT;
	DBuf<int> cInfo;
	DBuf<long long> pcgTiming;
	// the barrier of every cooperative kernel on the stream (k_pcg2/3/4, k_coarse_dense, k_dense_chol, peer all-reduce), zeroed in init()
	DBuf<GridBar> gridBar;
	PinnedArena arena;
	double curLambda = 0;           // damping of the solve being launched
	// reductions
	DBuf<double> chiPartial, scalePartialL, scalePartialP, chiSq;
	// edge levels (cuba_levels.cuh); allocated by the first level call, so that a run without levels keeps its footprint
	bool lvOn = false;             // levels used since the last set_problem: e_om0 holds the caller's omega, lvLevel the levels
	long long lvIncluded = 0;      // edges at level 0: all ranks' (under CUBA_DRY_SHARD this rank's own: its optimize() sees no other)
	DBuf<T> e_om0;                 // landmark-major omega as set_problem scattered it, before the mask
	DBuf<unsigned char> lvLevel;   // [E] in edge-id order; a rank reads and writes its own edges only
	DBuf<int> lvPartial;
	DBuf<double> lvCount;
	// optimize_landmarks: per-CTA counts, the per-round totals | status word (one read-back), the device list's marks
	DBuf<int> lrPartial, lrMark;
	DBuf<double> lrTotal;
	DBuf<Scalars> dScal;
	Scalars* hScal = nullptr;   // pinned
	DBuf<double> flushBuf;
	std::vector<std::pair<int, std::pair<cudaEvent_t, cudaEvent_t>>> profEvents;
	std::vector<cudaEvent_t> eventPool;
	cudaEvent_t joinIn = nullptr, joinOut = nullptr;   // the caller's stream -> the engine's, and back (on_caller_stream)

	~Engine() override
	{
		DevGuard guard(devOrdinal);
		if (stream) cudaStreamSynchronize(stream);
		p5Peer.close(rank); uPeer.close(rank);
		for (auto& pe : profEvents) { cudaEventDestroy(pe.second.first); cudaEventDestroy(pe.second.second); }
		for (auto ev : eventPool) cudaEventDestroy(ev);
		if (joinIn) cudaEventDestroy(joinIn);
		if (joinOut) cudaEventDestroy(joinOut);
		if (hScal) cudaFreeHost(hScal);
		if (hMeta) cudaFreeHost(hMeta);
		if (wt.host) cudaFreeHost(wt.host);
		if (stream) cudaStreamDestroy(stream);
		if (comm && g_nccl.CommDestroy) g_nccl.CommDestroy(comm);
	}

	int init()
	{
		int ndev = 0;
		cudaError_t e = cudaGetDeviceCount(&ndev);
		if (e != cudaSuccess || ndev <= 0)
			return fail(CUBA_ERR_CUDA, std::string("no CUDA device available (") + cudaGetErrorString(e) + "); this library has no CPU fallback");
		if (cfg.device >= 0) CUDA_TRY(cudaSetDevice(cfg.device));
		int dev = 0;
		CUDA_TRY(cudaGetDevice(&dev));
		devOrdinal = dev;
		CUDA_TRY(cudaDeviceGetAttribute(&numSMs, cudaDevAttrMultiProcessorCount, dev));
		CUDA_TRY(cudaDeviceGetAttribute(&smemMax, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
		CUDA_TRY(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
		CUDA_TRY(cudaEventCreateWithFlags(&joinIn, cudaEventDisableTiming)); CUDA_TRY(cudaEventCreateWithFlags(&joinOut, cudaEventDisableTiming));
		CUDA_TRY(cudaMallocHost((void**)&hScal, sizeof(Scalars)));
		memset(hScal, 0, sizeof(Scalars));
		CUDA_TRY(dScal.alloc(1));
		CUDA_TRY(cudaMemsetAsync(dScal.p, 0, sizeof(Scalars), stream));
		CUDA_TRY(gridBar.alloc(1)); CUDA_TRY(cudaMemsetAsync(gridBar.p, 0, sizeof(GridBar), stream));
		// for every coarse matrix k_coarse_invert takes (launch_coarse_setup), whichever solver it belongs to
		CUDA_TRY(cudaFuncSetAttribute(k_coarse_invert<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)coarse_invert_smem(PCG4_MAXAGG1)));
		int rc = stage_choice(cfg, sizeof(T) == 8, stages); if (rc) return rc;
		if (stages.jh4) {
			const void*& fn = wt.fn; size_t& smem = wt.smem;
#define JH4_PICK(MB, NS, ...) { fn = (const void*)jh4::k_linearize_landmark4<MB, NS, __VA_ARGS__>; smem = (size_t)NS * jh4::WARPS * sizeof(jh4::StageOf<MB, NS>); }
			if (stages.mixed) JH4_PICK(4, 2, 0, true)
			else if (stages.jh4Stages == 3) JH4_PICK(4, 3, 0)
			else if (stages.jh4MinB == 4) JH4_PICK(4, 2, 0)
			else if (stages.jh4MinB == 5) JH4_PICK(5, 2, 0)
			else JH4_PICK(6, 2, 0)
			CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
		}
		return CUBA_OK;
	}

	// ---- profile helpers: CUDA events on the launching stream, resolved lazily ----------------------
	cudaEvent_t newEvent()
	{
		cudaEvent_t ev;
		if (!eventPool.empty()) { ev = eventPool.back(); eventPool.pop_back(); return ev; }
		cudaEventCreate(&ev);
		return ev;
	}
	struct ProfScope {
		Engine* e; int item; cudaEvent_t a, b;
		ProfScope(Engine* e_, int item_) : e(e_), item(item_) { a = e->newEvent(); b = e->newEvent(); cudaEventRecord(a, e->stream); }
		~ProfScope() { cudaEventRecord(b, e->stream); e->profEvents.push_back({ item, { a, b } }); }
	};
	void resolveProfile()
	{
		cudaStreamSynchronize(stream);
		for (auto& pe : profEvents) {
			float ms = 0;
			if (cudaEventElapsedTime(&ms, pe.second.first, pe.second.second) == cudaSuccess) prof[pe.first] += 1e-3 * ms;
			eventPool.push_back(pe.second.first); eventPool.push_back(pe.second.second);
		}
		profEvents.clear();
	}

	RobustParams rkParams() const
	{
		RobustParams r;
		for (int i = 0; i < 2; i++) { r.type[i] = rk_type[i]; r.delta[i] = rk_delta[i]; }
		return r;
	}

	// Runs f on the engine's stream after the work the caller has queued on `caller` so far, and orders the caller's later work after
	// f's: an event each way (none for NULL or the engine's own stream).  Neither synchronises, so a capture of `caller` takes the
	// engine's work as a fork and a join of the graph.
	template <class F>
	int on_caller_stream(cudaStream_t caller, F&& f)
	{
		const bool join = caller && caller != stream;
		if (join) { CUDA_TRY(cudaEventRecord(joinIn, caller)); CUDA_TRY(cudaStreamWaitEvent(stream, joinIn, 0)); }
		const int rc = f();
		if (join) { CUDA_TRY(cudaEventRecord(joinOut, stream)); CUDA_TRY(cudaStreamWaitEvent(caller, joinOut, 0)); }
		return rc;
	}

	// ---- collectives (landmark-sharded runs) ----------------------------------------------------------
	int allreduce(void* buf, size_t count, bool isT)
	{
		if (world <= 1 || !comm) return CUBA_OK;      // (!comm: CUBA_DRY_SHARD diagnosis, one shard of a sharded run timed on one GPU)
		const int dt = isT ? (sizeof(T) == 8 ? NCCL_FLOAT64 : NCCL_FLOAT32) : NCCL_FLOAT64;
		const int rc = g_nccl.AllReduce(buf, buf, count, dt, NCCL_SUM, comm, stream);
		if (rc != 0) return fail(CUBA_ERR_COMM, std::string("ncclAllReduce failed: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?"));
		return CUBA_OK;
	}

	// ---- problem upload -------------------------------------------------------------------------------
	// ---- problem upload ----------------------------------------------------------------------------
	// The caller's flat fp64 arrays go to the device as they are; one kernel packs them into the padded records
	// (pose [8] = q,t,pad; cam [8]; Xw [4]) of the initial state and of both working buffers.
	DBuf<double> rawQ, rawT, rawC, rawX;
	int upload_state(const double* q, const double* t, const double* c, const double* X)
	{
		const int Pall = S.Pall, Lall = S.Lall;
		CUDA_TRY(rawQ.upload(q, 4 * (size_t)Pall, stream)); CUDA_TRY(rawT.upload(t, 3 * (size_t)Pall, stream));
		CUDA_TRY(rawX.upload(X, 3 * (size_t)Lall, stream));
		if (c) CUDA_TRY(rawC.upload(c, 5 * (size_t)Pall, stream));
		return pack_state(rawQ.p, rawT.p, c ? rawC.p : nullptr, rawX.p);
	}
	// the padded records from flat fp64 arrays on the device, the engine's or the caller's (read in place); c == NULL keeps cam.
	// Allocates nothing once set_problem has sized the buffers.
	int pack_state(const double* q, const double* t, const double* c, const double* X)
	{
		const int Pall = S.Pall, Lall = S.Lall;
		CUDA_TRY(pose0.alloc(8 * (size_t)Pall)); CUDA_TRY(Xw0.alloc(4 * (size_t)Lall));
		for (int b = 0; b < 2; b++) { CUDA_TRY(pose[b].alloc(8 * (size_t)Pall)); CUDA_TRY(Xw[b].alloc(4 * (size_t)Lall)); }
		if (c) CUDA_TRY(cam.alloc(8 * (size_t)Pall));
		const int n = std::max(Pall, Lall);
		if (n > 0) {
			k_pack_state<T><<<(n + 255) / 256, 256, 0, stream>>>(q, t, c, X, Pall, Lall,
				pose0.p, pose[0].p, pose[1].p, c ? cam.p : nullptr, Xw0.p, Xw[0].p, Xw[1].p);
			launches++;
			CUDA_TRY(cudaGetLastError());
		}
		// no synchronisation here: set_problem / set_state synchronise before they return to the caller
		return CUBA_OK;
	}

	// set_problem wall-clock marks (CUBA_SETUP_TIMING=1 prints them)
	std::vector<std::pair<const char*, std::chrono::steady_clock::time_point>> marks;
	void tmark(const char* name) { if (markOn) marks.push_back({ name, std::chrono::steady_clock::now() }); }
	bool markOn = false;
	int set_problem(const cuba_problem* p) override { return load_problem(p, false); }
	int set_problem_device(const cuba_problem* p, cudaStream_t caller) override
	{
		return on_caller_stream(caller, [&] { return load_problem(p, true); });
	}
	// set_problem from host arrays (dev = false) or from device arrays on the engine's device (dev = true: copied device to device,
	// the state read in place); everything else, structure reuse across both included, is one path
	int load_problem(const cuba_problem* p, bool dev)
	{
		markOn = getenv("CUBA_SETUP_TIMING") != nullptr; marks.clear(); tmark("start");
		if (!p) return fail(CUBA_ERR_INVALID, "set_problem: null problem");
		if (p->Pall < 0 || p->Lall < 0 || p->numP < 0 || p->numL < 0 || p->numP > p->Pall || p->numL > p->Lall || p->E2 < 0 || p->E3 < 0)
			return fail(CUBA_ERR_INVALID, "set_problem: invalid sizes");
		if ((p->Pall > 0 && (!p->q || !p->t || !p->cam)) || (p->Lall > 0 && !p->Xw) || (p->E2 > 0 && (!p->idx2 || !p->meas2 || !p->omega2)) ||
			(p->E3 > 0 && (!p->idx3 || !p->meas3 || !p->omega3)))
			return fail(CUBA_ERR_INVALID, "set_problem: null array with a non-zero count");
		// the cap, before any change; a pose-only system (no free landmark) never reaches the direct solver (k_solve_poses_only)
		if (linSolver == CUBA_SOLVER_DENSE_CHOLESKY && p->numP > dchol::MAX_POSES && p->numL > 0) return dense_cap_error(p->numP);
		if (dev && cfg.reserved[1] == 1)
			return fail(CUBA_ERR_INVALID, "set_problem_device: the host structure builder (reserved[1] = 1) reads host arrays; use set_problem");
		const auto t0 = std::chrono::steady_clock::now();
		lastPcgKernel = CUBA_PCG_KERNEL_NONE; p5.coarse.rebuilds = 0; bjRetries = 0;
		lvOn = false;      // every level back to 0: both paths below scatter the caller's omega unmasked
		// Same topology as the problem this engine already holds (sizes, fixed/free split and every (iP, iL) pair identical): only the
		// numbers changed -- the estimate after a previous optimize(), new measurements -- so every index structure, tile list,
		// product list and PCG partition on the device stays valid.  Upload the values and re-run the three kernels that scatter them.
		// Host lists are compared with the host copy of the held ones; device lists, or host lists after a device problem (no host
		// copy), on the device against g_idx2 / g_idx3, the flag read back with refresh_values' synchronisation -- when they differ,
		// the rebuild below overwrites everything the refresh wrote.
		if (structureReuse && reusable && haveProblem && cfg.reserved[1] != 1 && denseSolve == (linSolver == CUBA_SOLVER_DENSE_CHOLESKY) && same_sizes(p)) {
			const bool onDevice = dev || !lastIdxOnHost;
			bool same = onDevice || same_lists(p);
			if (same) {
				int rc = refresh_values(p, dev, onDevice, same); if (rc) return rc;
			}
			if (same) {
				if (!lastIdxOnHost && !dev) { keep_lists(p); lastIdxOnHost = true; }
				structureReuses++;
				prof[CUBA_PROF_BUILD_STRUCTURE] += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
				return CUBA_OK;
			}
		}
		haveProblem = false;
		reusable = false;
		hostStructureValid = false;
		shardBoundValid = false;
		int rc = (cfg.reserved[1] == 1) ? build_on_host(p) : build_on_gpu(p, dev);
		if (rc) return rc;
		tmark("structure built");
		rc = dev ? pack_state(p->q, p->t, p->cam, p->Xw) : upload_state(p->q, p->t, p->cam, p->Xw); if (rc) return rc;
		tmark("state uploaded");
		rc = alloc_system(); if (rc) return rc;
		CUDA_TRY(cudaStreamSynchronize(stream));
		tmark("alloc_system done");
		if (markOn) {
			for (size_t i = 1; i < marks.size(); i++)
				fprintf(stderr, "setup %-28s %8.3f ms\n", marks[i].first, 1e3 * std::chrono::duration<double>(marks[i].second - marks[i - 1].second).count());
			fprintf(stderr, "setup total %8.3f ms\n", 1e3 * std::chrono::duration<double>(marks.back().second - marks.front().second).count());
		}
		cur = 0; trialValid = false;
		forget_solves();
		resolveProfile();   // drop the events of earlier problems
		for (int i = 0; i < CUBA_PROF_NUM; i++) prof[i] = 0;
		const auto t1 = std::chrono::steady_clock::now();
		prof[CUBA_PROF_BUILD_STRUCTURE] += std::chrono::duration<double>(t1 - t0).count();
		haveProblem = true;
		if (cfg.reserved[1] != 1 && structureReuse) {
			if (dev) { lastIdx2.clear(); lastIdx3.clear(); }
			else keep_lists(p);
			lastIdxOnHost = !dev;
			const int sz[6] = { p->Pall, p->numP, p->Lall, p->numL, p->E2, p->E3 };
			memcpy(lastSizes, sz, sizeof(sz));
			reusable = true;
		}
		return CUBA_OK;
	}

	bool same_sizes(const cuba_problem* p) const
	{
		const int sz[6] = { p->Pall, p->numP, p->Lall, p->numL, p->E2, p->E3 };
		return memcmp(sz, lastSizes, sizeof(sz)) == 0;
	}
	bool same_lists(const cuba_problem* p) const
	{
		if (p->E2 > 0 && memcmp(p->idx2, lastIdx2.data(), sizeof(int32_t) * 2 * (size_t)p->E2) != 0) return false;
		if (p->E3 > 0 && memcmp(p->idx3, lastIdx3.data(), sizeof(int32_t) * 2 * (size_t)p->E3) != 0) return false;
		return true;
	}
	void keep_lists(const cuba_problem* p)
	{
		lastIdx2.assign(p->idx2, p->idx2 + 2 * (size_t)p->E2); lastIdx3.assign(p->idx3, p->idx3 + 2 * (size_t)p->E3);
	}

	// a raw problem array into the engine's buffer: uploaded from the host, or copied from the caller's device array
	template <typename U>
	cudaError_t put(DBuf<U>& b, const U* src, size_t n, bool dev) { return dev ? b.copy(src, n, stream) : b.upload(src, n, stream); }

	// set_problem on an unchanged topology: measurements, information values and the estimate go up (or across, dev), the edge streams
	// are re-scattered.  compare: the lists are first compared with the held ones on the device (host lists go up once for that);
	// same = false when they differ, and then nothing of the refresh counts (the caller rebuilds).
	int refresh_values(const cuba_problem* p, bool dev, bool compare, bool& same)
	{
		using namespace sgpu;
		const int E2 = p->E2, E3 = p->E3, eL = S.eLocal;
		if (compare) {
			const int32_t* i2 = p->idx2;
			const int32_t* i3 = p->idx3;
			if (!dev) {
				CUDA_TRY(cmpIdx2.upload(i2, 2 * (size_t)E2, stream)); CUDA_TRY(cmpIdx3.upload(i3, 2 * (size_t)E3, stream));
				i2 = cmpIdx2.p; i3 = cmpIdx3.p;
			}
			CUDA_TRY(cmpFlag.alloc(1));
			CUDA_TRY(cudaMemsetAsync(cmpFlag.p, 0, sizeof(int), stream));
			KLAUNCH(pio::k_idx_differ, 2 * ((long long)E2 + E3), i2, g_idx2.p, 2 * (long long)E2, i3, g_idx3.p, 2 * (long long)E3, cmpFlag.p);
		}
		CUDA_TRY(put(g_meas2, p->meas2, 2 * (size_t)E2, dev)); CUDA_TRY(put(g_meas3, p->meas3, 3 * (size_t)E3, dev));
		CUDA_TRY(put(g_om2, p->omega2, (size_t)E2, dev)); CUDA_TRY(put(g_om3, p->omega3, (size_t)E3, dev));
		int rc = dev ? pack_state(p->q, p->t, p->cam, p->Xw) : upload_state(p->q, p->t, p->cam, p->Xw); if (rc) return rc;
		KLAUNCH(k_edge_stream<T>, eL, g_keyS.p, g_valS.p, g_ff.p, g_hplG.p, savedKBeg, eL, S.hplBase, E2, g_meas2.p, g_om2.p, g_meas3.p, g_om3.p,
			e_user.p, e_ip.p, e_il.p, e_hpl.p, e_mx.p, e_my.p, e_mz.p, e_om.p);
		KLAUNCH(k_pose_stream<T>, eL, g_psrc.p, posePtr.p, S.numP, eL, e_ip.p, e_il.p, e_mx.p, e_my.p, e_mz.p, e_om.p, p_il.p, p_mx.p, p_my.p, p_mz.p, p_om.p);
		rc = jh4_emit(); if (rc) return rc;
		int differ = 0;
		if (compare) {
			g_d2hBytes += (long long)sizeof(differ);
			CUDA_TRY(cudaMemcpyAsync(&differ, cmpFlag.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
		}
		CUDA_TRY(cudaStreamSynchronize(stream));      // the caller's buffers are free again
		same = differ == 0;
		if (!same) return CUBA_OK;
		cur = 0; trialValid = false;
		forget_solves();
		resolveProfile();
		for (int i = 0; i < CUBA_PROF_NUM; i++) prof[i] = 0;
		return CUBA_OK;
	}

	// host structure builder (cuba_structure.cpp): reference path for the GPU builder, cfg.reserved[1] == 1
	int build_on_host(const cuba_problem* p)
	{
		const char* err = "";
		if (!build_structure(p->Pall, p->numP, p->Lall, p->numL, p->E2, p->idx2, p->E3, p->idx3, rank, world, stages.tileSize, S, &err))
			return fail(CUBA_ERR_INVALID, err);
		hostStructureValid = true;
		const int eL = S.eLocal;
		std::vector<T> mx(eL), my(eL), mz(eL), om(eL);
		for (int e = 0; e < eL; e++) {
			const int u = S.order[e];
			if (u < S.E2) { mx[e] = (T)p->meas2[2 * (size_t)u]; my[e] = (T)p->meas2[2 * (size_t)u + 1]; mz[e] = T(0); om[e] = (T)p->omega2[u]; }
			else { const size_t k = (size_t)(u - S.E2); mx[e] = (T)p->meas3[3 * k]; my[e] = (T)p->meas3[3 * k + 1]; mz[e] = (T)p->meas3[3 * k + 2]; om[e] = (T)p->omega3[k]; }
		}
		CUDA_TRY(e_mx.upload(mx, stream)); CUDA_TRY(e_my.upload(my, stream)); CUDA_TRY(e_mz.upload(mz, stream)); CUDA_TRY(e_om.upload(om, stream));
		CUDA_TRY(e_ip.upload(S.e_ip, stream)); CUDA_TRY(e_il.upload(S.e_il, stream)); CUDA_TRY(e_hpl.upload(S.e_hpl, stream));
		CUDA_TRY(e_user.upload(S.order, stream));
		CUDA_TRY(lmPtr.upload(S.lmPtr, stream)); CUDA_TRY(tilePtr.upload(S.lmPtr, stream));
		CUDA_TRY(tileLm.upload(S.tileLm, stream)); CUDA_TRY(hplLm.upload(S.hplLm, stream));
		const size_t nPe = S.p_src.size();
		std::vector<T> qx(nPe), qy(nPe), qz(nPe), qo(nPe);
		for (size_t k = 0; k < nPe; k++) { const int e = S.p_src[k]; qx[k] = mx[e]; qy[k] = my[e]; qz[k] = mz[e]; qo[k] = om[e]; }
		CUDA_TRY(p_mx.upload(qx, stream)); CUDA_TRY(p_my.upload(qy, stream)); CUDA_TRY(p_mz.upload(qz, stream)); CUDA_TRY(p_om.upload(qo, stream));
		CUDA_TRY(p_il.upload(S.p_il, stream)); CUDA_TRY(posePtr.upload(S.posePtr, stream));
		CUDA_TRY(prodPtr.upload(S.prodPtr, stream)); CUDA_TRY(prodI.upload(S.prodI, stream)); CUDA_TRY(prodJ.upload(S.prodJ, stream));
		CUDA_TRY(blkRow.upload(S.blkRow, stream)); CUDA_TRY(blkCol.upload(S.blkCol, stream));
		CUDA_TRY(u2f.upload(S.u2f, stream)); CUDA_TRY(u2fT.upload(S.u2fT, stream));
		CUDA_TRY(fRowPtr.upload(S.fRowPtr, stream)); CUDA_TRY(fColInd.upload(S.fColInd, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));   // host staging vectors die here
		ntiles = (int)S.tileLm.size() - 1;
		return CUBA_OK;
	}

	// ---- device structure builder (cuba_structure_gpu.cuh) ------------------------------------------------
	DBuf<int> g_idx2, g_idx3, g_val, g_valS, g_ff, g_hplG, g_lmPtrG, g_hplRowInd, g_hplLmG, g_edge2Hpl, g_hplColPtr, g_hscRowPtr;
	DBuf<int> g_pval, g_pvalS, g_pi, g_pj, g_head, g_blkId, g_cnt, g_off, g_fval, g_fvalS, g_pkeyVal, g_psrc;
	DBuf<double> g_meas2, g_meas3, g_om2, g_om3;
	DBuf<unsigned long long> g_key, g_keyS, g_pkey, g_pkeyS, g_fkey, g_fkeyS;
	DBuf<unsigned int> g_k32, g_k32S;
	DBuf<char> cubTmp;
	DBuf<sgpu::Meta> g_meta;
	sgpu::Meta* hMeta = nullptr;
	bool hostStructureValid = false;
	// structure reuse across set_problem calls (repeated local BA on an unchanged graph): the last problem's index lists
	std::vector<int32_t> lastIdx2, lastIdx3;
	bool lastIdxOnHost = true;    // lastIdx2 / lastIdx3 hold the lists (false after a set_problem_device: g_idx2 / g_idx3 only)
	DBuf<int> cmpIdx2, cmpIdx3, cmpFlag;   // the device comparison of refresh_values: host lists, "some word differs"
	int lastSizes[6] = { -1, -1, -1, -1, -1, -1 };
	int savedKBeg = 0;
	bool reusable = false;      // the device structures of the last problem are complete and were built on the device
	int shardBound[9] = { 0 };    // first landmark of every rank's shard
	bool shardBoundValid = false;

	template <typename K>
	int sortPairs(K* kin, K* kout, int* vin, int* vout, int n, int endBit)
	{
		if (n <= 0) return CUBA_OK;
		size_t bytes = 0;
		CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, bytes, kin, kout, vin, vout, n, 0, endBit, stream));
		CUDA_TRY(cubTmp.alloc(bytes));
		CUDA_TRY(cub::DeviceRadixSort::SortPairs(cubTmp.p, bytes, kin, kout, vin, vout, n, 0, endBit, stream));
		launches += 4;
		return CUBA_OK;
	}
	int exclusiveSum(const int* in, int* out, int n)
	{
		if (n <= 0) return CUBA_OK;
		size_t bytes = 0;
		CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, stream));
		CUDA_TRY(cubTmp.alloc(bytes));
		CUDA_TRY(cub::DeviceScan::ExclusiveSum(cubTmp.p, bytes, in, out, n, stream));
		launches += 2;
		return CUBA_OK;
	}
	int fetchMeta()
	{
		if (!hMeta) CUDA_TRY(cudaMallocHost((void**)&hMeta, sizeof(sgpu::Meta)));
		CUDA_TRY(cudaMemcpyAsync(hMeta, g_meta.p, sizeof(sgpu::Meta), cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		if (hMeta->error == 1) return fail(CUBA_ERR_INVALID, "build_structure: edge index out of range");
		if (hMeta->error == 2) return fail(CUBA_ERR_INVALID, "build_structure: edge with both ends fixed");
		if (hMeta->error == 3) return fail(CUBA_ERR_INVALID, "build_structure: free landmark without edges (the reference's initialize() drops such vertices)");
		return CUBA_OK;
	}

	int build_on_gpu(const cuba_problem* p, bool dev)
	{
		using namespace sgpu;
		S = Structure();
		const int Pall = p->Pall, numP = p->numP, Lall = p->Lall, numL = p->numL, E2 = p->E2, E3 = p->E3, E = E2 + E3;
		S.Pall = Pall; S.numP = numP; S.Lall = Lall; S.numL = numL; S.E2 = E2; S.E3 = E3; S.E = E;
		// raw problem -> device (the only bulk H2D traffic of set_problem besides the state; none from device arrays)
		CUDA_TRY(put(g_idx2, p->idx2, 2 * (size_t)E2, dev)); CUDA_TRY(put(g_idx3, p->idx3, 2 * (size_t)E3, dev));
		CUDA_TRY(put(g_meas2, p->meas2, 2 * (size_t)E2, dev)); CUDA_TRY(put(g_meas3, p->meas3, 3 * (size_t)E3, dev));
		CUDA_TRY(put(g_om2, p->omega2, (size_t)E2, dev)); CUDA_TRY(put(g_om3, p->omega3, (size_t)E3, dev));
		CUDA_TRY(g_meta.alloc(1));
		CUDA_TRY(cudaMemsetAsync(g_meta.p, 0, sizeof(Meta), stream));
		// 1. canonical (iL, iP, edge id) order
		CUDA_TRY(g_key.alloc(E)); CUDA_TRY(g_keyS.alloc(E)); CUDA_TRY(g_val.alloc(E)); CUDA_TRY(g_valS.alloc(E));
		KLAUNCH(k_make_keys, E, E2, g_idx2.p, E3, g_idx3.p, Pall, numP, Lall, numL, g_key.p, g_val.p, g_meta.p);
		int rc = sortPairs(g_key.p, g_keyS.p, g_val.p, g_valS.p, E, 32 + bits_for((unsigned long long)std::max(Lall, 1))); if (rc) return rc;
		CUDA_TRY(g_lmPtrG.alloc((size_t)Lall + 1));
		KLAUNCH(k_ptr_from_high, Lall + 1, g_keyS.p, E, Lall, g_lmPtrG.p);
		KLAUNCH(k_check_nonempty, numL, g_lmPtrG.p, numL, g_meta.p);
		// 2. Hpl blocks = free-free edges in canonical order
		CUDA_TRY(g_ff.alloc(E)); CUDA_TRY(g_hplG.alloc(E));
		KLAUNCH(k_flag_freefree, E, g_keyS.p, E, numP, numL, g_ff.p);
		rc = exclusiveSum(g_ff.p, g_hplG.p, E); if (rc) return rc;
		k_shard_meta<<<1, 32, 0, stream>>>(g_lmPtrG.p, Lall, E, rank, world, g_ff.p, g_hplG.p, g_meta.p);
		launches++;
		CUDA_TRY(cudaGetLastError());
		tmark("queued to sync 1");
		rc = fetchMeta(); if (rc) return rc;                                   // sync point 1
		tmark("sync 1");
		S.nhpl = hMeta->nhpl; S.lmBeg = hMeta->lmBeg; S.lmEnd = hMeta->lmEnd; S.eLocal = hMeta->kEnd - hMeta->kBeg;
		S.hplBase = hMeta->hplBase; S.nhplLocal = hMeta->hplEnd - hMeta->hplBase;
		for (int r = 0; r < 9; r++) shardBound[r] = hMeta->bounds[r];
		shardBoundValid = true;
		const int kBeg = hMeta->kBeg, kEnd = hMeta->kEnd, eL = S.eLocal, nhpl = S.nhpl;
		savedKBeg = kBeg;
		CUDA_TRY(g_hplRowInd.alloc(nhpl)); CUDA_TRY(g_hplLmG.alloc(nhpl)); CUDA_TRY(g_edge2Hpl.alloc(E)); CUDA_TRY(g_hplColPtr.alloc((size_t)numL + 1));
		KLAUNCH(k_hpl_global, E, g_keyS.p, g_valS.p, g_ff.p, g_hplG.p, E, g_hplRowInd.p, g_hplLmG.p, g_edge2Hpl.p);
		KLAUNCH(k_hpl_colptr, numL + 1, g_lmPtrG.p, g_hplG.p, E, numL, nhpl, g_hplColPtr.p);
		// 3. landmark-major stream of the shard, tiles
		CUDA_TRY(e_user.alloc(eL)); CUDA_TRY(e_ip.alloc(eL)); CUDA_TRY(e_il.alloc(eL)); CUDA_TRY(e_hpl.alloc(eL));
		CUDA_TRY(e_mx.alloc(eL)); CUDA_TRY(e_my.alloc(eL)); CUDA_TRY(e_mz.alloc(eL)); CUDA_TRY(e_om.alloc(eL));
		KLAUNCH(k_edge_stream<T>, eL, g_keyS.p, g_valS.p, g_ff.p, g_hplG.p, kBeg, eL, S.hplBase, E2, g_meas2.p, g_om2.p, g_meas3.p, g_om3.p,
			e_user.p, e_ip.p, e_il.p, e_hpl.p, e_mx.p, e_my.p, e_mz.p, e_om.p);
		CUDA_TRY(lmPtr.alloc((size_t)Lall + 1));
		KLAUNCH(k_local_lmptr, Lall + 1, g_lmPtrG.p, Lall, kBeg, kEnd, lmPtr.p);
		CUDA_TRY(hplLm.alloc(S.nhplLocal));
		if (S.nhplLocal > 0) CUDA_TRY(cudaMemcpyAsync(hplLm.p, g_hplLmG.p + S.hplBase, sizeof(int) * (size_t)S.nhplLocal, cudaMemcpyDeviceToDevice, stream));
		CUDA_TRY(tilePtr.alloc((size_t)numL + 2));
		KLAUNCH(k_tile_ptr, numL + 2, lmPtr.p, numL, eL, tilePtr.p);
		const int tb = std::min(S.lmBeg, numL), te = std::min(S.lmEnd, numL) + (S.lmEnd > numL ? 1 : 0);
		// windows a little shorter than the CTA so that the tail of a tile's last landmark usually still fits one chunk
		const int window = stages.tileSize - 16;
		const int nt = (eL + window - 1) / window;
		CUDA_TRY(tileLm.alloc((size_t)nt + 1));
		KLAUNCH(k_tiles, nt + 1, tilePtr.p, tb, te, window, nt, tileLm.p);
		ntiles = nt;
		// 4. pose-major stream (free poses only)
		CUDA_TRY(g_k32.alloc(eL)); CUDA_TRY(g_k32S.alloc(eL)); CUDA_TRY(g_pval.alloc(eL)); CUDA_TRY(g_psrc.alloc(eL));
		KLAUNCH(k_pose_keys, eL, e_ip.p, eL, numP, g_k32.p, g_pval.p);
		rc = sortPairs(g_k32.p, g_k32S.p, g_pval.p, g_psrc.p, eL, bits_for((unsigned long long)numP)); if (rc) return rc;
		CUDA_TRY(posePtr.alloc((size_t)numP + 1));
		KLAUNCH(k_ptr_from_u32, numP + 1, g_k32S.p, eL, numP, posePtr.p);
		CUDA_TRY(p_il.alloc(eL)); CUDA_TRY(p_mx.alloc(eL)); CUDA_TRY(p_my.alloc(eL)); CUDA_TRY(p_mz.alloc(eL)); CUDA_TRY(p_om.alloc(eL));
		KLAUNCH(k_pose_stream<T>, eL, g_psrc.p, posePtr.p, numP, eL, e_ip.p, e_il.p, e_mx.p, e_my.p, e_mz.p, e_om.p, p_il.p, p_mx.p, p_my.p, p_mz.p, p_om.p);
		// 5. block products keyed by destination block, + one dummy per diagonal
		CUDA_TRY(g_cnt.alloc((size_t)nhpl + 1)); CUDA_TRY(g_off.alloc((size_t)nhpl + 1));
		CUDA_TRY(cudaMemsetAsync(g_cnt.p, 0, sizeof(int) * ((size_t)nhpl + 1), stream));
		KLAUNCH(k_prod_count, nhpl, g_hplLmG.p, g_hplColPtr.p, g_hplRowInd.p, nhpl, g_cnt.p, g_meta.p);
		rc = exclusiveSum(g_cnt.p, g_off.p, nhpl + 1); if (rc) return rc;
		long long nmul = 0;
		{
			int last = 0;
			CUDA_TRY(cudaMemcpyAsync(&last, g_off.p + nhpl, sizeof(int), cudaMemcpyDeviceToHost, stream));
			tmark("queued to sync 2");
			CUDA_TRY(cudaStreamSynchronize(stream));                              // sync point 2
			tmark("sync 2");
			nmul = last;
		}
		S.nmul = nmul;
		const long long N = nmul + numP;
		if (N > 0x7fffffffLL) return fail(CUBA_ERR_INVALID, "build_structure: more than 2^31 block products");
		S.nmulLocal = N;
		CUDA_TRY(g_pkey.alloc((size_t)N)); CUDA_TRY(g_pkeyS.alloc((size_t)N)); CUDA_TRY(g_pkeyVal.alloc((size_t)N)); CUDA_TRY(g_pvalS.alloc((size_t)N));
		CUDA_TRY(g_pi.alloc((size_t)N)); CUDA_TRY(g_pj.alloc((size_t)N));
		KLAUNCH(k_prod_emit, nhpl, g_hplLmG.p, g_hplColPtr.p, g_hplRowInd.p, g_off.p, nhpl, S.lmBeg, S.lmEnd, S.hplBase, g_pkey.p, g_pkeyVal.p, g_pi.p, g_pj.p);
		KLAUNCH(k_prod_diag, numP, numP, nmul, g_pkey.p, g_pkeyVal.p, g_pi.p, g_pj.p);
		rc = sortPairs(g_pkey.p, g_pkeyS.p, g_pkeyVal.p, g_pvalS.p, (int)N, 32 + bits_for((unsigned long long)std::max(numP, 1))); if (rc) return rc;
		CUDA_TRY(g_head.alloc((size_t)N + 1)); CUDA_TRY(g_blkId.alloc((size_t)N + 1));
		KLAUNCH(k_heads, N, g_pkeyS.p, (int)N, g_head.p);
		rc = exclusiveSum(g_head.p, g_blkId.p, (int)N); if (rc) return rc;
		k_nblk<<<1, 32, 0, stream>>>(g_head.p, g_blkId.p, (int)N, g_meta.p);
		launches++;
		tmark("queued to sync 3");
		rc = fetchMeta(); if (rc) return rc;                                   // sync point 3
		tmark("sync 3");
		const int nblk = hMeta->nblk;
		S.nblk = nblk;
		S.repeatedPairs = hMeta->repeats != 0;
		CUDA_TRY(blkRow.alloc(nblk)); CUDA_TRY(blkCol.alloc(nblk)); CUDA_TRY(prodPtr.alloc((size_t)nblk + 1));
		CUDA_TRY(prodI.alloc((size_t)N)); CUDA_TRY(prodJ.alloc((size_t)N));
		KLAUNCH(k_blocks, N + 1, g_pkeyS.p, g_pvalS.p, g_head.p, g_blkId.p, g_pi.p, g_pj.p, (int)N, blkRow.p, blkCol.p, prodPtr.p, prodI.p, prodJ.p);
		CUDA_TRY(g_hscRowPtr.alloc((size_t)numP + 1));
		KLAUNCH(k_rowptr_from_rows, numP + 1, blkRow.p, nblk, numP, g_hscRowPtr.p);
		int* dLocalCount = nullptr;
		if (world > 1) {
			// the sorted list holds every rank's products (the block numbering must be global); a destination's warp would walk all of
			// them and skip the foreign ones -- the Schur kernel then does not speed up with the rank count (measured: a 1/8
			// shard of the 10 M-edge graph took over a third of the time of the whole).  Keep the local products and the diagonal placeholders only.
			CUDA_TRY(g_head.alloc((size_t)N + 1)); CUDA_TRY(g_blkId.alloc((size_t)N + 1));
			KLAUNCH(k_local_flag, N + 1, prodI.p, prodJ.p, (int)N, g_head.p);
			rc = exclusiveSum(g_head.p, g_blkId.p, (int)N + 1); if (rc) return rc;
			KLAUNCH(k_compact_products, N, prodI.p, prodJ.p, g_head.p, g_blkId.p, (int)N, g_pi.p, g_pj.p);
			KLAUNCH(k_remap_ptr, nblk + 1, g_blkId.p, nblk, prodPtr.p);
			CUDA_TRY(cudaMemcpyAsync(prodI.p, g_pi.p, sizeof(int) * (size_t)N, cudaMemcpyDeviceToDevice, stream));
			CUDA_TRY(cudaMemcpyAsync(prodJ.p, g_pj.p, sizeof(int) * (size_t)N, cudaMemcpyDeviceToDevice, stream));
			dLocalCount = g_blkId.p + N;
		}
		// 6. symmetric-full BSR for the PCG
		const int nfull = 2 * nblk - numP;
		S.nfull = nfull;
		CUDA_TRY(g_fkey.alloc(2 * (size_t)nblk)); CUDA_TRY(g_fkeyS.alloc(2 * (size_t)nblk)); CUDA_TRY(g_fval.alloc(2 * (size_t)nblk)); CUDA_TRY(g_fvalS.alloc(2 * (size_t)nblk));
		KLAUNCH(k_full_entries, nblk, blkRow.p, blkCol.p, nblk, numP, g_fkey.p, g_fval.p);
		rc = sortPairs(g_fkey.p, g_fkeyS.p, g_fval.p, g_fvalS.p, 2 * nblk, 32 + bits_for((unsigned long long)std::max(numP, 1))); if (rc) return rc;
		CUDA_TRY(fColInd.alloc(nfull)); CUDA_TRY(u2f.alloc(nblk)); CUDA_TRY(u2fT.alloc(nblk)); CUDA_TRY(fRowPtr.alloc((size_t)numP + 1));
		KLAUNCH(k_full_finish, nfull, g_fkeyS.p, g_fvalS.p, nfull, blkRow.p, blkCol.p, fColInd.p, u2f.p, u2fT.p);
		KLAUNCH(k_ptr_from_high, numP + 1, g_fkeyS.p, nfull, numP, fRowPtr.p);
		// the PCG partition is computed on the host from the (small) full pattern
		S.fRowPtr.resize((size_t)numP + 1); S.fColInd.resize(nfull);
		g_d2hBytes += (long long)(sizeof(int) * ((size_t)numP + 1 + nfull));
		CUDA_TRY(cudaMemcpyAsync(S.fRowPtr.data(), fRowPtr.p, sizeof(int) * ((size_t)numP + 1), cudaMemcpyDeviceToHost, stream));
		if (nfull > 0) CUDA_TRY(cudaMemcpyAsync(S.fColInd.data(), fColInd.p, sizeof(int) * (size_t)nfull, cudaMemcpyDeviceToHost, stream));
		int localCount = (int)N;
		if (dLocalCount) CUDA_TRY(cudaMemcpyAsync(&localCount, dLocalCount, sizeof(int), cudaMemcpyDeviceToHost, stream));
		tmark("queued to sync 4");
		CUDA_TRY(cudaStreamSynchronize(stream));                                  // sync point 4
		tmark("sync 4");
		S.nmulLocal = localCount;
		return CUBA_OK;
	}

	// host copies of the index structures, only for the debug getters
	int ensureHostStructure()
	{
		if (hostStructureValid) return CUBA_OK;
		auto dl = [&](std::vector<int>& dst, const int* src, size_t n) -> cudaError_t {
			dst.resize(n);
			return n ? cudaMemcpyAsync(dst.data(), src, sizeof(int) * n, cudaMemcpyDeviceToHost, stream) : cudaSuccess;
		};
		CUDA_TRY(dl(S.hplColPtr, g_hplColPtr.p, (size_t)S.numL + 1)); CUDA_TRY(dl(S.hplRowInd, g_hplRowInd.p, S.nhpl));
		CUDA_TRY(dl(S.edge2Hpl, g_edge2Hpl.p, S.E)); CUDA_TRY(dl(S.hscRowPtr, g_hscRowPtr.p, (size_t)S.numP + 1));
		CUDA_TRY(dl(S.hscColInd, blkCol.p, S.nblk)); CUDA_TRY(dl(S.u2f, u2f.p, S.nblk)); CUDA_TRY(dl(S.u2fT, u2fT.p, S.nblk));
		CUDA_TRY(cudaStreamSynchronize(stream));
		hostStructureValid = true;
		return CUBA_OK;
	}

	int alloc_system()
	{
		const int eL = S.eLocal;
		const size_t nP = S.numP, nL = S.numL;
		// Hpp | bp | (chi2 slot) and Hsc | bsc are single allocations: one collective each in landmark-sharded runs
		CUDA_TRY(Hpp.alloc(42 * nP + 2)); bp.alias(Hpp.p + 36 * nP, 6 * nP);
		CUDA_TRY(Hll.alloc(9 * nL)); CUDA_TRY(bl.alloc(3 * nL));
		if (stages.mixed) { CUDA_TRY(HplF.alloc(20 * (size_t)std::max(S.nhplLocal, 1))); CUDA_TRY(Hpl.alloc(1)); }
		else CUDA_TRY(Hpl.alloc(18 * (size_t)S.nhplLocal));
		CUDA_TRY(invHll.alloc(9 * nL));
		CUDA_TRY(fVal.alloc(36 * (size_t)S.nfull + 6 * nP)); bsc.alias(fVal.p + 36 * (size_t)S.nfull, 6 * nP);
		// k_schur3 serves a tensor-pipe request the structure cannot (no products on this rank; a repeated (pose, landmark) pair: its bsc
		// term rides on every product of a diagonal destination).  upperReduce follows the request, so every rank joins one collective.
		useSchur5 = stages.schur5 && S.numP > 0 && S.numL > 0 && ntiles > 0 && S.eLocal > 0 && S.nmulLocal > 0 && !S.repeatedPairs;
		upperReduce = world > 1 && !stages.schur5 && S.numP > 0 && S.numL > 0;
		if (upperReduce) {
			uCount = 36 * (size_t)S.nblk + 6 * nP;
			const size_t need = peer_signal_offset(uCount) + 64;          // + the signal block of the peer all-reduce
			if (!uVal.p || need > uVal.cap) {
				if (uPeer.mappedFor) { CUDA_TRY(cudaStreamSynchronize(stream)); uPeer.close(rank); }
				CUDA_TRY(uVal.alloc(std::max(need, (size_t)1 << 18)));
				CUDA_TRY(cudaMemsetAsync(uVal.p, 0, sizeof(T) * uVal.cap, stream));
				uEpoch = 0;
			}
			bsc.alias(uVal.p + 36 * (size_t)S.nblk, 6 * nP);
			// map the peers' buffers; the signal block must sit at the same offset everywhere (it does: uCount is global)
			uPeerOk = false;
			if (!getenv("CUBA_NCCL_HSC") && comm) {
				// signals of an earlier problem may sit at another offset: start from a clean block (all ranks do, in lockstep)
				CUDA_TRY(cudaMemsetAsync(uVal.p + peer_signal_offset(uCount), 0, sizeof(T) * 64, stream));
				uEpoch = 0;
				int rcx = allreduce(&dScal.p->v[7], 1, false); if (rcx) return rcx;          // nobody signals into a block that is being cleared
				bool ok = false;
				rcx = ipcExchange((void*)uVal.p, uPeer, ok); if (rcx) return rcx;
				uPeerOk = ok;
			}
		}
		CUDA_TRY(xp.alloc(6 * nP)); CUDA_TRY(xl.alloc(3 * nL));
		// landmarks outside this rank's shard keep zero Hll/bl/xl (they are never touched locally)
		if (nL) CUDA_TRY(cudaMemsetAsync(Hll.p, 0, sizeof(T) * 9 * nL, stream));
		if (nL) CUDA_TRY(cudaMemsetAsync(bl.p, 0, sizeof(T) * 3 * nL, stream));
		if (nL) CUDA_TRY(cudaMemsetAsync(xl.p, 0, sizeof(T) * 3 * nL, stream));
		if (nP) CUDA_TRY(cudaMemsetAsync(xp.p, 0, sizeof(T) * 6 * nP, stream));
		if (nP) CUDA_TRY(cudaMemsetAsync(Hpp.p, 0, sizeof(T) * 36 * nP, stream));
		if (nP) CUDA_TRY(cudaMemsetAsync(bp.p, 0, sizeof(T) * 6 * nP, stream));
		if (useSchur5) { int rc = setup_schur5(); if (rc) return rc; }
		else if (S.nmulLocal > 0) {
			CUDA_TRY(prodL.alloc((size_t)S.nmulLocal));
			KLAUNCH(schur3::k_prod_landmark, S.nmulLocal, prodI.p, hplLm.p, (int)S.nmulLocal, prodL.p);
		}
		tmark("alloc + Schur setup queued");
		if (stages.jh4) { int rc = setup_jh4(); if (rc) return rc; }
		tmark("jh4 queued");
		// the solver's setup: no PCG partition or plan for the direct solver (its need lists may not fit, and nothing reads them)
		denseSolve = linSolver == CUBA_SOLVER_DENSE_CHOLESKY;
		p3.pcg3 = false; p4.ok = false; p5Ok = false;          // what a structure before this one prepared
		if (denseSolve) {
			if (S.numP > 0 && S.numL > 0) { int rc = setup_dense(); if (rc) return rc; }
			else release_dense();
		}
		else {
			release_dense();                                                   // up to 1 GB of tiles nothing reads any more
			pick = pcg_choice();
			if (S.numP > 0) { int rc = setup_pcg3(); if (rc) return rc; }        // host-heavy: overlaps the warp-tile kernels queued above
			if (S.numP > 0 && pick.p4) { int rc = setup_pcg4(hostPP); if (rc) return rc; }
			if (S.numP > 0 && S.numL > 0 && pick.p5) { int rc = setup_pcg5(); if (rc) return rc; }
		}
		tmark("pcg partition (host)");
		if (stages.jh4) { int rc = setup_jh4_finish(); if (rc) return rc; }
		tmark("jh4 finish");
		nPoseBlocks = (S.numP + RED_BLOCK - 1) / RED_BLOCK;
		nChiBlocks = std::max(1, std::min((eL + RED_BLOCK - 1) / RED_BLOCK, numSMs * 8));
		CUDA_TRY(chiPartial.alloc((size_t)std::max(std::max(ntiles, nChiBlocks), wt.grid) + 1));
		CUDA_TRY(scalePartialL.alloc((size_t)std::max(ntiles, (S.numL + RED_BLOCK - 1) / RED_BLOCK) + 1));
		CUDA_TRY(scalePartialP.alloc((size_t)nPoseBlocks + 1));
		CUDA_TRY(chiSq.alloc((size_t)S.E));
		return CUBA_OK;
	}

	int set_state(const double* q, const double* t, const double* X) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "set_state before set_problem");
		const int rc = upload_state(q, t, nullptr, X); if (rc) return rc;
		CUDA_TRY(cudaStreamSynchronize(stream));      // the caller's buffers are free again
		trialValid = false;
		return CUBA_OK;
	}

	int set_state_device(const double* q, const double* t, const double* X, cudaStream_t caller) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "set_state before set_problem");
		return on_caller_stream(caller, [&] { trialValid = false; return pack_state(q, t, nullptr, X); });
	}

	int reset_state() override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "reset_state before set_problem");
		for (int b = 0; b < 2; b++) {
			CUDA_TRY(cudaMemcpyAsync(pose[b].p, pose0.p, sizeof(T) * 8 * (size_t)S.Pall, cudaMemcpyDeviceToDevice, stream));
			CUDA_TRY(cudaMemcpyAsync(Xw[b].p, Xw0.p, sizeof(T) * 4 * (size_t)S.Lall, cudaMemcpyDeviceToDevice, stream));
		}
		trialValid = false;
		return CUBA_OK;
	}
	int flush_l2() override
	{
		const size_t flushN = (size_t)40 << 20;
		CUDA_TRY(flushBuf.alloc(flushN));
		k_fill<<<numSMs * 8, 256, 0, stream>>>(flushBuf.p, flushN, 1.0);
		launches++;
		CUDA_TRY(cudaGetLastError());
		return CUBA_OK;
	}

	int get_sizes(cuba_sizes* o) const override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "get_sizes before set_problem");
		o->Pall = S.Pall; o->numP = S.numP; o->Lall = S.Lall; o->numL = S.numL; o->E2 = S.E2; o->E3 = S.E3;
		o->nhpl = S.nhpl; o->nblk = S.nblk; o->nmul = (int32_t)S.nmul; o->nblk_full = S.nfull;
		return CUBA_OK;
	}

	// ---- launches --------------------------------------------------------------------------------------
	ChiArgs<T> chiArgs(int buf)
	{
		ChiArgs<T> a;
		a.pose = pose[buf]; a.cam = cam; a.Xw = Xw[buf];
		a.mx = e_mx; a.my = e_my; a.mz = e_mz; a.om = e_om; a.ip = e_ip; a.il = e_il;
		a.E = S.eLocal; a.rk = rkParams(); a.chiPartial = chiPartial;
		return a;
	}

	int launch_linearize_landmark()
	{
		if (ntiles <= 0) return CUBA_OK;
		if (stages.jh4) return launch_jh4();
		LinLmArgs<T> a;
		a.pose = pose[cur]; a.cam = cam; a.Xw = Xw[cur];
		a.mx = e_mx; a.my = e_my; a.mz = e_mz; a.om = e_om; a.ip = e_ip; a.il = e_il; a.hpl = e_hpl;
		a.lmPtr = tilePtr; a.tileLm = tileLm; a.numP = S.numP; a.numL = S.numL;
		a.Hpl = Hpl; a.Hll = Hll; a.bl = bl; a.chiPartial = chiPartial; a.rk = rkParams();
		if (stages.tileSize == 128 && stages.minBlocks >= 6) k_linearize_landmark<T, 128, 6><<<ntiles, 128, 0, stream>>>(a);
		else if (stages.tileSize == 128) k_linearize_landmark<T, 128, 4><<<ntiles, 128, 0, stream>>>(a);
		else if (stages.minBlocks >= 3) k_linearize_landmark<T, 256, 3><<<ntiles, 256, 0, stream>>>(a);
		else k_linearize_landmark<T, 256, 2><<<ntiles, 256, 0, stream>>>(a);
		launches++;
		CUDA_TRY(cudaGetLastError());
		return CUBA_OK;
	}
	// The warp-tile pass over wt.  -DCUBA_JH4_DEBUG (tools/jh4_dbg.sh): CUBA_JH4_DBG launches an instrumented instance of the shape
	// instead of wt.fn, except under mixed precision; with bit 3 the phase counters of the fourth launch go to stderr.
	int launch_jh4()
	{
		if constexpr (sizeof(T) == 8) {
			if (wt.ntiles <= 0) return CUBA_OK;
			jh4::Args b;
			b.pose = pose[cur]; b.cam = cam; b.Xw = Xw[cur];
			b.rec = wt.rec; b.tile = wt.tile; b.tilePose = wt.tilePose; b.tilePieces = wt.tilePieces; b.pieceCount = wt.pieceCount; b.ntiles = wt.ntiles; b.numL = S.numL;
			b.Hpl = Hpl; b.HplF = stages.mixed ? HplF.p : nullptr; b.Hll = Hll; b.bl = bl; b.bigPartial = wt.bigPartial; b.chiPartial = chiPartial; b.rk = rkParams();
			const void* fn = wt.fn; size_t smem = wt.smem;
#ifdef CUBA_JH4_DEBUG
			int dbg = getenv("CUBA_JH4_DBG") ? atoi(getenv("CUBA_JH4_DBG")) : 0;
			if (stages.jh4Stages == 3) { switch (dbg) { case 1: JH4_PICK(4, 3, 1) break; case 2: JH4_PICK(4, 3, 2) break; case 4: JH4_PICK(4, 3, 4) break; case 6: JH4_PICK(4, 3, 6) break;
				case 7: JH4_PICK(4, 3, 7) break; case 8: JH4_PICK(4, 3, 8) break; case 15: JH4_PICK(4, 3, 15) break; default: dbg = 0; } }
			else { switch (dbg) { case 8: JH4_PICK(5, 2, 8) break; case 7: JH4_PICK(5, 2, 7) break; default: dbg = 0; } }
			if (stages.mixed) { fn = wt.fn; smem = wt.smem; }
			if (fn != wt.fn) CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
#endif
			void* kargs[] = { (void*)&b };
			CUDA_TRY(cudaLaunchKernel(fn, dim3(wt.grid), dim3(jh4::WARPS * 32), kargs, smem, stream));
#ifdef CUBA_JH4_DEBUG
			if (dbg & 8) {
				const int nw = wt.grid * jh4::WARPS;
				std::vector<double> h(11 * (size_t)nw);
				cudaMemcpyAsync(h.data(), wt.bigPartial.p, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, stream);
				cudaStreamSynchronize(stream);
				double acc[8] = { 0 };
				for (int w = 0; w < nw; w++) for (int i = 0; i < 8; i++) acc[i] += h[8 * (size_t)w + i];
				static int once = 0;
				if (once++ == 3) {
					const char* nm[8] = { "cpasync_wait", "mbar_wait", "lds_inputs", "math+hpl_staging", "fence+bulk_store", "wait_read+issue", "reduce+stores", "rotate(descr)" };
					double tot = 0; for (int i = 0; i < 8; i++) tot += acc[i];
					for (int i = 0; i < 8; i++) fprintf(stderr, "jh4 phase %-18s %9.0f cycles/warp  %5.1f %%\n", nm[i], acc[i] / nw, 100 * acc[i] / tot);
					fprintf(stderr, "jh4 total %9.0f cycles/warp, %d warps, %d tiles\n", tot / nw, nw, wt.ntiles);
					double s0 = 1e300, s1 = 0, l0 = 1e300, l1 = 0, e0 = 1e300, e1 = 0;
					for (int w = 0; w < nw; w++) {
						const double* g = h.data() + 8 * (size_t)nw + 3 * (size_t)w;
						s0 = std::min(s0, g[0]); s1 = std::max(s1, g[0]); l0 = std::min(l0, g[1]); l1 = std::max(l1, g[1]); e0 = std::min(e0, g[2]); e1 = std::max(e1, g[2]);
					}
					fprintf(stderr, "jh4 globaltimer (ns, rel. first start): start %.0f..%.0f  loop entry %.0f..%.0f  loop exit %.0f..%.0f\n", 0.0, s1 - s0, l0 - s0, l1 - s0, e0 - s0, e1 - s0);
				}
			}
#endif
			launches++;
			CUDA_TRY(cudaGetLastError());
		}
		return CUBA_OK;
	}
	int launch_linearize_pose()
	{
		if (S.numP <= 0) return CUBA_OK;
		LinPoseArgs<T> a;
		a.pose = pose[cur]; a.cam = cam; a.Xw = Xw[cur];
		a.mx = p_mx; a.my = p_my; a.mz = p_mz; a.om = p_om; a.il = p_il; a.posePtr = posePtr;
		a.Hpp = Hpp; a.bp = bp; a.rk = rkParams();
		k_linearize_pose<T><<<S.numP, POSE_BLOCK, 0, stream>>>(a);
		launches++;
		CUDA_TRY(cudaGetLastError());
		return CUBA_OK;
	}
	// sums chiPartial[0..n) (+ optional two more arrays) into dScal->v[slot..slot+2]
	int launch_sum(const double* p0, int n0, const double* p1, int n1, const double* p2, int n2, int slot)
	{
		k_sum_partials<<<1, RED_BLOCK, 0, stream>>>(p0, n0, p1, n1, p2, n2, &dScal.p->v[slot]);
		launches++;
		CUDA_TRY(cudaGetLastError());
		return CUBA_OK;
	}
	int fetchScalars()
	{
		g_d2hBytes += (long long)sizeof(Scalars);
		CUDA_TRY(cudaMemcpyAsync(hScal, dScal.p, sizeof(Scalars), cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		return CUBA_OK;
	}

	int stage_linearize(double* chi) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "linearize before set_problem");
		{
			ProfScope ps(this, CUBA_PROF_BUILD_SYSTEM);
			int rc = launch_linearize_landmark(); if (rc) return rc;
			rc = launch_linearize_pose(); if (rc) return rc;
			rc = launch_sum(chiPartial, ntiles <= 0 ? 0 : stages.jh4 ? wt.grid : ntiles, nullptr, 0, nullptr, 0, 0); if (rc) return rc;
			if (world > 1) {
				// ONE collective: Hpp | bp | chi2 are contiguous (the chi2 partial rides in the slot behind bp)
				if constexpr (sizeof(T) == 8) {
					T* slot = Hpp.p + 42 * (size_t)S.numP;
					CUDA_TRY(cudaMemcpyAsync(slot, &dScal.p->v[0], sizeof(double), cudaMemcpyDeviceToDevice, stream));
					rc = allreduce(Hpp.p, 42 * (size_t)S.numP + 1, true); if (rc) return rc;
					CUDA_TRY(cudaMemcpyAsync(&dScal.p->v[0], slot, sizeof(double), cudaMemcpyDeviceToDevice, stream));
				} else {
					if (S.numP > 0) { rc = allreduce(Hpp.p, 42 * (size_t)S.numP, true); if (rc) return rc; }
					rc = allreduce(&dScal.p->v[0], 1, false); if (rc) return rc;
				}
			}
		}
		int rc = fetchScalars(); if (rc) return rc;
		if (chi) *chi = hScal->v[0];
		return CUBA_OK;
	}

	int stage_chi2(double* chi) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "chi2 before set_problem");
		int rc = launch_chi2(cur, 0); if (rc) return rc;
		rc = fetchScalars(); if (rc) return rc;
		if (chi) *chi = hScal->v[0];
		return CUBA_OK;
	}

	int launch_chi2(int buf, int slot, bool reduce = true)
	{
		ProfScope ps(this, CUBA_PROF_COMPUTE_ERROR);
		if (S.eLocal > 0) {
			k_chi2<T><<<nChiBlocks, RED_BLOCK, 0, stream>>>(chiArgs(buf));
			launches++;
			CUDA_TRY(cudaGetLastError());
		}
		int rc = launch_sum(chiPartial, S.eLocal > 0 ? nChiBlocks : 0, nullptr, 0, nullptr, 0, slot); if (rc) return rc;
		if (world > 1 && reduce) { rc = allreduce(&dScal.p->v[slot], 1, false); if (rc) return rc; }
		return CUBA_OK;
	}

	int stage_max_diagonal(double* md) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "max_diagonal before set_problem");
		CUDA_TRY(cudaMemsetAsync(&dScal.p->maxdiag, 0, sizeof(unsigned long long), stream));
		const int n = S.numP * 6 + S.numL * 3;
		if (n > 0) {
			const int grid = std::max(1, std::min((n + 255) / 256, numSMs * 4));
			k_max_diagonal<T><<<grid, 256, 0, stream>>>(Hpp, S.numP, Hll, S.numL, &dScal.p->maxdiag);
			launches++;
			CUDA_TRY(cudaGetLastError());
		}
		if (world > 1) {
			const int rcn = comm ? g_nccl.AllReduce(&dScal.p->maxdiag, &dScal.p->maxdiag, 1, NCCL_FLOAT64, NCCL_MAX, comm, stream) : 0;
			if (rcn != 0) return fail(CUBA_ERR_COMM, "ncclAllReduce(max) failed");
		}
		int rc = fetchScalars(); if (rc) return rc;
		double m;
		memcpy(&m, &hScal->maxdiag, sizeof(double));
		if (md) *md = m;
		return CUBA_OK;
	}

	int launch_schur(T lambda)
	{
		ProfScope ps(this, CUBA_PROF_SCHUR_COMPLEMENT);
		if (useSchur5) return launch_schur5(lambda);
		{
			// the inverses of this rank's landmarks only (nobody reads the others here)
			const int l0 = std::min(S.lmBeg, S.numL), l1 = std::min(S.lmEnd, S.numL);
			if (l1 > l0) {
				k_inv_hll<T><<<(l1 - l0 + 255) / 256, 256, 0, stream>>>(Hll.p + 9 * (size_t)l0, l1 - l0, lambda, invHll.p + 9 * (size_t)l0);
				launches++;
				CUDA_TRY(cudaGetLastError());
			}
		}
		if (S.numP > 0 && S.numL > 0) {
			int rc = stages.mixed ? launch_schur3(HplF.p, lambda) : launch_schur3(Hpl.p, lambda); if (rc) return rc;
			if (upperReduce) {
				// upper blocks | bsc: one collective of half the bytes, then both triangles are filled locally
				static const bool timing = getenv("CUBA_SCHUR_TIMING") != nullptr;      // diagnosis: split of the stage, printed by rank 0
				cudaEvent_t ev[3];
				if (timing) { for (auto& e : ev) cudaEventCreate(&e); cudaEventRecord(ev[0], stream); }
				rc = uPeerOk ? launch_peer_allreduce() : allreduce(uVal.p, 36 * (size_t)S.nblk + 6 * (size_t)S.numP, true); if (rc) return rc;
				if (timing) cudaEventRecord(ev[1], stream);
				KLAUNCH(schur3::k_expand_upper<T>, 36LL * S.nblk, uVal.p, u2f.p, u2fT.p, blkRow.p, blkCol.p, S.nblk, fVal.p);
				if (timing) {
					cudaEventRecord(ev[2], stream); cudaEventSynchronize(ev[2]);
					float a1 = 0, a2 = 0; cudaEventElapsedTime(&a1, ev[0], ev[1]); cudaEventElapsedTime(&a2, ev[1], ev[2]);
					static int count = 0;
					if (rank == 0 && (count++ % 16) == 8) fprintf(stderr, "schur split: all-reduce (%s) %.3f ms, expand %.3f ms, %zu elements\n", uPeerOk ? "peer" : "nccl", a1, a2, uCount);
					for (auto& e : ev) cudaEventDestroy(e);
				}
			}
			else if (world > 1) {
				rc = allreduce(fVal.p, 36 * (size_t)S.nfull + 6 * (size_t)S.numP, true); if (rc) return rc;   // Hsc | bsc: one buffer
			}
		}
		return CUBA_OK;
	}
	// k_schur3 on Hpl blocks of type HT: T, or float under mixed precision
	template <typename HT>
	int launch_schur3(const HT* hpl, T lambda)
	{
		schur3::Args<T, HT> a;
		a.Hpl = hpl; a.invHll = invHll; a.bl = bl; a.Hpp = Hpp; a.bp = bp;
		a.prodPtr = prodPtr; a.prodI = prodI; a.prodJ = prodJ; a.prodL = prodL;
		a.blkRow = blkRow; a.blkCol = blkCol; a.u2f = u2f; a.u2fT = u2fT; a.nblk = S.nblk;
		a.lambda = lambda; a.addDiag = rank == 0 ? 1 : 0; a.fVal = fVal; a.bsc = bsc; a.uVal = upperReduce ? uVal.p : nullptr;
		schur3::k_schur3<T, HT><<<(S.nblk + schur3::WARPS - 1) / schur3::WARPS, schur3::WARPS * 32, 0, stream>>>(a);
		launches++;
		CUDA_TRY(cudaGetLastError());
		return CUBA_OK;
	}
	// the Schur complement on the tensor pipe (s5): the products of each (tile, destination) segment, then one reduction per block
	int launch_schur5(T lambda)
	{
		if constexpr (sizeof(T) == 8) {
			schur5::Args sa;
			sa.Hpl = Hpl; sa.Hll = Hll; sa.bl = bl; sa.info = s5.tileInfo; sa.hplLm = hplLm; sa.tileSegPtr = s5.tileSegPtr; sa.segRec = s5.segRec; sa.off = s5.off;
			sa.p2i = s5.p2i; sa.p2j = s5.p2j; sa.numL = S.numL; sa.lambda = lambda; sa.invHll = invHll; sa.partial = s5.partial;
			schur5::k_schur_tiles_mma<<<s5.ntiles, schur5::WARPS * 32, sizeof(schur5::Smem), stream>>>(sa);
			launches++;
			CUDA_TRY(cudaGetLastError());
			schur5::ReduceArgs<T> ra;
			ra.partial = s5.partial; ra.destSegPtr = s5.destSegPtr; ra.Hpp = Hpp; ra.bp = bp;
			ra.blkRow = blkRow; ra.blkCol = blkCol; ra.u2f = u2f; ra.u2fT = u2fT; ra.nblk = S.nblk; ra.lambda = lambda;
			ra.addDiag = rank == 0 ? 1 : 0; ra.fVal = fVal; ra.bsc = bsc;
			schur5::k_schur_reduce<T><<<(S.nblk + 3) / 4, 128, 0, stream>>>(ra);
			launches++;
			CUDA_TRY(cudaGetLastError());
			if (world > 1) return allreduce(fVal.p, 36 * (size_t)S.nfull + 6 * (size_t)S.numP, true);   // Hsc | bsc: one buffer
		}
		return CUBA_OK;
	}

	// warp tiles of the J+H landmark pass (cuba_jh4.cuh): greedy packing by binary lifting, padded records, pose lists
	int setup_jh4()
	{
		wt.ntiles = 0; wt.grid = 0;
		const int lb = S.lmBeg, N = S.lmEnd - S.lmBeg;
		if (N <= 0 || S.eLocal <= 0) return CUBA_OK;
		int K = 1;
		while ((1LL << K) <= (long long)N) K++;
		CUDA_TRY(wt.levels.alloc((size_t)K * ((size_t)N + 1)));
		CUDA_TRY(wt.start.alloc((size_t)N + 1)); CUDA_TRY(wt.pieces.alloc((size_t)N + 1)); CUDA_TRY(wt.base.alloc((size_t)N + 1));
		CUDA_TRY(wt.flag.alloc(1));
		CUDA_TRY(cudaMemsetAsync(wt.flag.p, 0, sizeof(int), stream));
		KLAUNCH(jh4::k_next, N + 1, lmPtr.p, lb, N, wt.levels.p);
		for (int k = 1; k < K; k++)
			KLAUNCH(jh4::k_lift, N + 1, wt.levels.p + (size_t)(k - 1) * ((size_t)N + 1), N, wt.levels.p + (size_t)k * ((size_t)N + 1));
		KLAUNCH(jh4::k_starts, N + 1, wt.levels.p, K, N, lmPtr.p, lb, wt.start.p, wt.pieces.p, wt.flag.p);
		int rc = exclusiveSum(wt.pieces.p, wt.base.p, N + 1); if (rc) return rc;
		if (!wt.host) CUDA_TRY(cudaMallocHost((void**)&wt.host, 2 * sizeof(int)));
		CUDA_TRY(cudaMemcpyAsync(&wt.host[0], wt.base.p + N, sizeof(int), cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaMemcpyAsync(&wt.host[1], wt.flag.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
		wt.pending = true;
		return CUBA_OK;
	}
	// second half of the warp-tile setup: the host work of the PCG setups runs between the two halves, overlapping the kernels above
	int setup_jh4_finish()
	{
		if (!wt.pending) return CUBA_OK;
		wt.pending = false;
		CUDA_TRY(cudaStreamSynchronize(stream));
		const int big = wt.host[1], nt = wt.ntiles = wt.host[0];
		if (nt <= 0) return CUBA_OK;
		CUDA_TRY(wt.tile.alloc(nt)); CUDA_TRY(wt.rec.alloc(nt)); CUDA_TRY(wt.tilePose.alloc(32 * (size_t)nt)); CUDA_TRY(wt.tilePieces.alloc(nt)); CUDA_TRY(wt.pieceCount.alloc(nt));
		CUDA_TRY(cudaMemsetAsync(wt.pieceCount.p, 0, sizeof(int) * (size_t)nt, stream));
		CUDA_TRY(wt.bigPartial.alloc(std::max<size_t>(big ? 12 * (size_t)nt : 12, 11 * (size_t)numSMs * 6 * jh4::WARPS)));
		int rc = jh4_emit(); if (rc) return rc;
		wt.grid = std::max(1, std::min((nt + jh4::WARPS - 1) / jh4::WARPS, numSMs * stages.jh4MinB));
		return CUBA_OK;
	}
	// the warp-tile records from the landmark-major edge streams: at setup, and whenever a refresh or the level mask rewrites them
	int jh4_emit()
	{
		if constexpr (sizeof(T) == 8) {
			if (wt.ntiles <= 0) return CUBA_OK;
			const int lb = S.lmBeg, N = S.lmEnd - S.lmBeg;
			KLAUNCH(jh4::k_emit, (long long)N * 32, wt.start.p, wt.pieces.p, wt.base.p, N, lmPtr.p, lb, wt.levels.p,
				e_mx.p, e_my.p, e_mz.p, e_om.p, e_ip.p, e_il.p, e_hpl.p, wt.tile.p, wt.rec.p, wt.tilePose.p, wt.tilePieces.p);
		}
		return CUBA_OK;
	}

	// landmark tiles of the Schur stage (its own, larger ones: windows of schur5::WINDOW edges), (tile, destination) segments of
	// the block products, segment records and operand offsets of k_schur_tiles_mma
	int setup_schur5()
	{
		using namespace schur5;
		const int N = (int)S.nmulLocal, nblk = S.nblk;
		const int tb5 = std::min(S.lmBeg, S.numL), te5 = std::min(S.lmEnd, S.numL) + (S.lmEnd > S.numL ? 1 : 0);
		const int nt = s5.ntiles = (S.eLocal + WINDOW - 1) / WINDOW;
		CUDA_TRY(s5.tileLm.alloc((size_t)nt + 1)); CUDA_TRY(s5.tileInfo.alloc((size_t)nt));
		KLAUNCH(sgpu::k_tiles, nt + 1, tilePtr.p, tb5, te5, WINDOW, nt, s5.tileLm.p);
		k_tile_info3<<<nt, 128, 0, stream>>>(tilePtr.p, s5.tileLm.p, e_ip.p, e_hpl.p, S.eLocal, S.nhplLocal, nt, s5.tileInfo.p);
		launches++;
		CUDA_TRY(cudaGetLastError());
		CUDA_TRY(s5.key.alloc(N)); CUDA_TRY(s5.keyS.alloc(N)); CUDA_TRY(s5.val.alloc(N)); CUDA_TRY(s5.valS.alloc(N));
		CUDA_TRY(s5.head.alloc(N)); CUDA_TRY(s5.segId.alloc(N)); CUDA_TRY(s5.counts.alloc(1));
		KLAUNCH(k_keys, N, prodPtr.p, nblk, prodI.p, N, s5.tileInfo.p, nt, s5.key.p, s5.val.p);
		int rc = sortPairs(s5.key.p, s5.keyS.p, s5.val.p, s5.valS.p, N, 64); if (rc) return rc;
		KLAUNCH(k_heads, N, s5.keyS.p, N, s5.head.p);
		rc = exclusiveSum(s5.head.p, s5.segId.p, N); if (rc) return rc;
		k_counts<<<1, 32, 0, stream>>>(s5.keyS.p, s5.head.p, s5.segId.p, N, s5.counts.p);
		launches++;
		Counts hc;
		CUDA_TRY(cudaMemcpyAsync(&hc, s5.counts.p, sizeof(hc), cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		const int nseg = hc.nseg, nvalid = hc.nvalid;
		CUDA_TRY(s5.segStart.alloc((size_t)nseg + 1)); CUDA_TRY(s5.segTile.alloc(nseg)); CUDA_TRY(s5.segDest.alloc(nseg));
		CUDA_TRY(s5.key3.alloc(nseg)); CUDA_TRY(s5.key3S.alloc(nseg)); CUDA_TRY(s5.val3.alloc(nseg)); CUDA_TRY(s5.val3S.alloc(nseg));
		CUDA_TRY(s5.segRank.alloc(nseg)); CUDA_TRY(s5.rankDest.alloc(nseg));
		CUDA_TRY(s5.tileSegPtr.alloc((size_t)nt + 1)); CUDA_TRY(s5.destSegPtr.alloc((size_t)nblk + 1));
		CUDA_TRY(s5.p2i.alloc(N)); CUDA_TRY(s5.p2j.alloc(N));
		KLAUNCH(k_segments, N + 1, s5.keyS.p, s5.valS.p, s5.head.p, s5.segId.p, prodI.p, prodJ.p, N, nseg, nvalid,
			s5.segStart.p, s5.segTile.p, s5.segDest.p, s5.p2i.p, s5.p2j.p, s5.key3.p, s5.val3.p);
		KLAUNCH(k_ptr_from_field, nt + 1, s5.segTile.p, nseg, nt, s5.tileSegPtr.p);
		rc = sortPairs(s5.key3.p, s5.key3S.p, s5.val3.p, s5.val3S.p, nseg, 32 + sgpu::bits_for((unsigned long long)std::max(nblk, 1))); if (rc) return rc;
		KLAUNCH(k_rank, nseg, s5.key3S.p, s5.val3S.p, nseg, s5.segRank.p, s5.rankDest.p);
		KLAUNCH(k_ptr_from_field, nblk + 1, s5.rankDest.p, nseg, nblk, s5.destSegPtr.p);
		CUDA_TRY(s5.partial.alloc((size_t)PW * std::max(nseg, 1)));
		CUDA_TRY(s5.segRec.alloc((size_t)std::max(nseg, 1)));
		KLAUNCH(k_seg_records, nseg, s5.segStart.p, s5.segDest.p, s5.segRank.p, s5.segTile.p, blkRow.p, blkCol.p, s5.tileInfo.p, s5.p2i.p, s5.p2j.p, nseg, s5.segRec.p);
		CUDA_TRY(s5.off.alloc((size_t)std::max(nvalid, 1)));
		KLAUNCH(k_prod_offsets, nvalid, s5.segStart.p, s5.segTile.p, s5.tileInfo.p, s5.p2i.p, s5.p2j.p, nseg, nvalid, s5.off.p);
		CUDA_TRY(cudaFuncSetAttribute(k_schur_tiles_mma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Smem)));
		return CUBA_OK;
	}

	// ---- the PCG kernel of a solve -------------------------------------------------------------------------------------------------
	// The choice of a structure: the runs to prepare besides the block-Jacobi one, k_pcg5 distributed over the ranks or not, and the
	// steps of a solve before and after the policy turned two-level (tlActive) and of the block-Jacobi retry of a breakdown.  A step
	// runs k_pcg5 (two-level or block-Jacobi) when it has a plan, else k_pcg4 when it is prepared, else block-Jacobi k_pcg3 -- k_pcg2
	// beyond k_pcg3's rows per CTA or when asked for (pcg2).
	// cfg.reserved[0] (pcg_variant): 0 (also 7: never distributed, 8: distributed at any size) automatic -- block-Jacobi (k_pcg5 when
	// distributed, k_pcg3 otherwise) until the policy turns two-level, then k_pcg5, or k_pcg4 without a k_pcg5 plan; 5: always
	// two-level k_pcg5; 6: always block-Jacobi k_pcg5; 3: always k_pcg4; 4: always k_pcg3; 2: k_pcg2.  k_pcg4 is prepared where it can
	// be asked for: explicitly, by the fp32 engine, or as the fallback for systems beyond k_pcg5's 85 rows per CTA.
	struct PcgStep { bool p5 = false, twoLevel = false, p4 = false; };
	struct PcgChoice { bool p4 = false, p5 = false, dist = false, pcg2 = false; PcgStep first, later, retry; };
	PcgChoice pick;                      // of the current structure (alloc_system)
	PcgChoice pcg_choice() const
	{
		const int m = cfg.reserved[0], numP = S.numP;
		PcgChoice c;
		c.p4 = m == 3 || sizeof(T) != 8 || numP > 80 * numSMs * (world > 1 && numP >= 2048 ? world : 1);
		c.p5 = m != 2 && m != 3 && m != 4;
		c.dist = c.p5 && world > 1 && comm && m != 7 && (m == 8 || numP >= 2048);
		c.pcg2 = m == 2;
		if (m == 0 || m == 7 || m == 8) { c.first = c.retry = { c.dist, false, false }; c.later = { true, true, true }; }
		else if (m == 5) { c.first = c.later = { true, true, false }; c.retry = { true, false, false }; }
		else if (m == 6) c.first = c.later = c.retry = { true, false, false };
		else if (m == 3) c.first = c.later = { false, false, true };
		return c;
	}
	// dynamic shared memory of one CTA of k_pcg2 / k_pcg3 / k_pcg4: leave room for the static arrays (4.4 KB in k_pcg3)
	size_t pcg3_budget() const { return (size_t)smemMax > 8192 ? (size_t)smemMax - 6144 : 0; }
	// Row partition, need lists and shared-memory budget of the block-Jacobi solve (p3).
	int setup_pcg3()
	{
		const int numP = S.numP;
		const size_t budget = pcg3_budget();
		const size_t matBytes = (size_t)S.nfull * (36 * sizeof(T) + 4);
		int G = std::max((numP + 7) / 8, (int)((matBytes + budget - 1) / std::max<size_t>(budget, 1)));
		G = std::max(1, std::min(G, std::min(numSMs, numP)));
		// row partition, need lists, block-local column positions: cuba_structure.cpp (CPU-tested)
		PcgPartition& PP = hostPP;                     // kept: k_pcg4 and k_pcg5's plan start from the same partition
		build_pcg_partition(numP, S.nfull, S.fRowPtr, S.fColInd, G, PP);
		const int needMax = PP.needMax, blkMax = PP.blkMax, maxRows = PP.maxRows;
		const size_t needBytes = pcg3_fixed_bytes(needMax, maxRows, sizeof(T));
		// k_pcg3 / k_pcg2 keep every needed column in shared memory and are the solver of last resort: without them no solve can run
		if (needBytes > budget) {
			const size_t perNeed = 12 * sizeof(T) + 8, rest = needBytes - (size_t)needMax * perNeed;
			const size_t fit = budget > rest ? (budget - rest) / perNeed : 0;
			return fail(CUBA_ERR_INVALID, "set_problem: a CTA of the block-Jacobi PCG needs " + std::to_string(needMax) + " columns of the reduced camera system ("
				+ std::to_string(needBytes) + " bytes of shared memory, " + std::to_string(budget) + " available: at most " + std::to_string(fit)
				+ " columns with " + std::to_string(maxRows) + " rows per CTA); the poses are too densely covisible for this engine");
		}
		p3.pcg3 = maxRows * 6 <= PCG3_BLOCK && 2 * G <= 2 * PCG3_BLOCK;   // k_pcg3: one (row,component) pair per thread, two partial words per thread
		size_t cap = budget > needBytes ? (budget - needBytes) / (36 * sizeof(T) + 4) : 0;
		cap = std::min<size_t>(cap, (size_t)blkMax);
		p3.G = G; p3.cap = (int)cap; p3.needMax = needMax; p3.maxRows = maxRows;
		p3.smem = (size_t)cap * 36 * sizeof(T) + needBytes + (size_t)cap * 4 + 16;
		CUDA_TRY(cudaFuncSetAttribute(k_pcg2<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p3.smem));
		CUDA_TRY(cudaFuncSetAttribute(k_pcg3<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p3.smem));
		CUDA_TRY(p3.flags.alloc(2 * (2 * 6 * (size_t)numP) + 2 * (2 * PCG3_REPL * 2 * (size_t)G) + 2));
		int perSM = 0;
		CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, k_pcg2<T>, PCG2_BLOCK, p3.smem));
		if (perSM < 1) return fail(CUBA_ERR_CUDA, "k_pcg2 cannot be resident with the requested shared memory");
		arena.reset();
		CUDA_TRY(p3.ctaRow.upload(PP.rows, stream, &arena)); CUDA_TRY(p3.needPtr.upload(PP.nptr, stream, &arena)); CUDA_TRY(p3.needCol.upload(PP.ncol, stream, &arena));
		CUDA_TRY(p3.local.upload(PP.local, stream, &arena));
		const size_t n6 = 6 * (size_t)numP;
		CUDA_TRY(fHat.alloc(36 * (size_t)S.nfull)); CUDA_TRY(p3.Linv.alloc(36 * (size_t)numP));
		CUDA_TRY(p3.R0.alloc(n6)); CUDA_TRY(p3.R1.alloc(n6)); CUDA_TRY(p3.S0.alloc(n6)); CUDA_TRY(p3.S1.alloc(n6));
		CUDA_TRY(p3.W0.alloc(n6)); CUDA_TRY(p3.W1.alloc(n6)); CUDA_TRY(p3.P.alloc(n6)); CUDA_TRY(p3.Y.alloc(n6));
		CUDA_TRY(p3.partial.alloc(4 * (size_t)G));
		tmark("  pcg2 partition + uploads");
		return CUBA_OK;
	}

	// k_pcg4 (p4) on the block-Jacobi partition PP: aggregates = groups of gs consecutive CTAs (at most PCG4_MAXAGG of them)
	int setup_pcg4(const PcgPartition& PP)
	{
		const int numP = S.numP, G = PP.G, needMax = PP.needMax, blkMax = PP.blkMax, maxRows = PP.maxRows;
		const size_t budget = pcg3_budget();
		// up to 74 aggregates, fewer with cfg.reserved[6] (37 or fewer: the coarse inverse of one CTA, k_coarse_invert)
		const int maxAgg = (cfg.reserved[6] > 0 && cfg.reserved[6] < PCG4_MAXAGG) ? cfg.reserved[6] : PCG4_MAXAGG;
		CoarsePartition CP;
		build_coarse_partition(numP, PP, maxAgg, CP);
		const int gs = CP.gs, A = CP.A, nc = 6 * A;
		p4.gs = gs; p4.maxNeedAgg = CP.maxNeedAgg;
		size_t fixed4 = (size_t)needMax * (12 * sizeof(T) + 8) + (size_t)maxRows * (6 * sizeof(T) + 8) + 8 + 2 * (size_t)nc * sizeof(T)
			+ (size_t)p4.maxNeedAgg * (6 * sizeof(T) + 4) + 64;
		// shared-memory priorities: all of A^ first, then Z^ of the needed columns, then the CTA's slices of the inverse coarse matrix
		const size_t matAll = (size_t)blkMax * (36 * sizeof(T) + 4);
		const size_t zhBytes = (size_t)needMax * 36 * sizeof(T);
		const size_t sliceBytes = (((size_t)p4.maxNeedAgg * 6 * nc + 1) & ~(size_t)1) * sizeof(float);
		p4.zhInSmem = budget >= fixed4 + matAll + zhBytes ? 1 : 0;
		if (p4.zhInSmem) fixed4 += zhBytes;
		p4.sliceInSmem = budget >= fixed4 + matAll + sliceBytes ? 1 : 0;
		if (p4.sliceInSmem) fixed4 += sliceBytes;
		size_t cap4 = budget > fixed4 ? (budget - fixed4) / (36 * sizeof(T) + 4) : 0;
		cap4 = std::min<size_t>(cap4, (size_t)blkMax);
		p4.cap = (int)cap4;
		p4.smem = (size_t)cap4 * (36 * sizeof(T) + 4) + fixed4;
		if (getenv("CUBA_PCG_VERBOSE")) fprintf(stderr, "pcg4: G %d A %d gs %d needMax %d maxRows %d blkMax %d maxNeedAgg %d zhInSmem %d sliceInSmem %d cap %d smem %zu\n",
			G, A, gs, needMax, maxRows, blkMax, p4.maxNeedAgg, p4.zhInSmem, p4.sliceInSmem, p4.cap, p4.smem);
		p4.ok = budget > fixed4 && nc + 64 <= PCG4_BLOCK && numP >= 2 * A;
		if (p4.ok) {
			CUDA_TRY(cudaFuncSetAttribute(k_pcg4<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p4.smem));
			int perSM4 = 0;
			CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM4, k_pcg4<T>, PCG4_BLOCK, p4.smem));
			if (perSM4 < 1) p4.ok = false;
		}
		if (!p4.ok) return CUBA_OK;
		// fine blocks of every coarse block (lower triangle), ascending -> fixed-order sums in k_coarse_assemble
		build_coarse_lists(numP, S.nfull, S.fRowPtr, S.fColInd, CP);
		int rc = p4.coarse.upload(CP, stream, &arena); if (rc) return rc;
		CUDA_TRY(cZx.alloc(36 * (size_t)numP)); CUDA_TRY(p4.Zhat.alloc(36 * (size_t)numP)); CUDA_TRY(cU.alloc(36 * (size_t)S.nfull));
		if (coarse_kernel(A) == CUBA_COARSE_KERNEL_DENSE) CUDA_TRY(cdT.alloc(cdense::scratch_doubles(A)));
		CUDA_TRY(p4.part.alloc(2 * (size_t)G * PCG4_PSTRIDE)); CUDA_TRY(cInfo.alloc(1));
		CUDA_TRY(cudaMemsetAsync(p4.part.p, 0, sizeof(double) * p4.part.n, stream));
		// (no synchronisation: the uploads above read the pinned arena, or were staged by the driver before returning)
		return CUBA_OK;
	}

	// two-level PCG: coarse basis, coarse matrix and its inverse, then the cooperative solve
	int launch_pcg4()
	{
		ProfScope ps(this, CUBA_PROF_DECOMP_NUMERICAL);
		KLAUNCH(k_coarse_basis<T>, S.numP, pose[cur].p, S.numP, cZx.p);
		const CoarseLevel& L = p4.coarse;
		int rc = coarse_refresh(p4.coarse, coarse_scratch(), cInfo.p); if (rc) return rc;     // slot 0 of cInfo
		Pcg4Args<T> b;
		b.base = pcg2_args(p3, p4.cap);
		b.Zx = cZx; b.Zhat = p4.Zhat; b.AcInv = L.AcInv; b.aggRow = L.aggRow; b.naPtr = L.naPtr; b.naList = L.naList;
		b.needAgg = L.needAgg; b.A = L.A; b.gs = p4.gs; b.maxNeedAgg = p4.maxNeedAgg; b.sliceInSmem = p4.sliceInSmem; b.zhInSmem = p4.zhInSmem; b.cpart = p4.part;
		b.timing = nullptr;
#ifdef CUBA_PCG_TIMING
		CUDA_TRY(pcgTiming.alloc(8 * (size_t)p3.G));
		b.timing = pcgTiming.p;
#endif
		void* args[] = { (void*)&b };
		CUDA_TRY(cudaLaunchCooperativeKernel((void*)k_pcg4<T>, dim3(p3.G), dim3(PCG4_BLOCK), args, p4.smem, stream));
		launches++;
		lastPcgTwoLevel = true;
		lastPcgKernel = CUBA_PCG_KERNEL_PCG4;
		return CUBA_OK;
	}
	bool lastPcgTwoLevel = false, tlActive = false;   // tlActive: the default solver's policy turned two-level (note_pcg_iters)
	bool forceBlockJacobi = false;   // retry of a trial whose two-level solve broke down
	// policy of the default solver: block-Jacobi (k_pcg3, the cheaper iteration) while it converges quickly, two-level (k_pcg4,
	// a dearer iteration but 2-8x fewer of them) once a block-Jacobi solve needed more than 100 iterations -- the count grows
	// as the LM damping falls.  The decision depends on iteration counts only, so runs stay bit-reproducible.
	void note_pcg_iters(int iters) { if (!lastPcgTwoLevel && iters > (cfg.reserved[5] > 0 ? cfg.reserved[5] : 100)) tlActive = true; }

	// the iteration cap and the squared relative tolerance of every PCG solve
	int pcg_max_iters() const { return cfg.pcg_max_iters > 0 ? cfg.pcg_max_iters : std::max(200, 40 * S.numP); }
	double pcg_tol2() const
	{
		const double tol = cfg.pcg_tol > 0 ? cfg.pcg_tol : (sizeof(T) == 8 ? 1e-11 : 1e-6);
		return tol * tol;
	}

	// the arguments of k_pcg2 / k_pcg3, and the block-Jacobi part of k_pcg4's, on R with capBlocks blocks of A^ in shared memory
	Pcg2Args<T> pcg2_args(const Pcg3Run& R, int capBlocks)
	{
		Pcg2Args<T> a;
		a.fRowPtr = fRowPtr; a.fColInd = fColInd; a.fLocal = R.local; a.fVal = fVal; a.fHat = fHat;
		a.ctaRow = R.ctaRow; a.needPtr = R.needPtr; a.needCol = R.needCol; a.b = bsc; a.numP = S.numP; a.Linv = R.Linv;
		a.R0 = R.R0; a.R1 = R.R1; a.S0 = R.S0; a.S1 = R.S1; a.W0 = R.W0; a.W1 = R.W1; a.P = R.P; a.Y = R.Y; a.x = xp;
		a.partial = R.partial; a.bar = gridBar; a.capBlocks = capBlocks; a.needMax = R.needMax; a.maxRows = R.maxRows;
		a.maxIters = pcg_max_iters(); a.tol2 = pcg_tol2();
		a.status = &dScal.p->pcg;
		return a;
	}

	// the block-Jacobi solve on p3: k_pcg3 (flag-synchronised exchange) or k_pcg2 (one grid barrier per iteration)
	int launch_pcg3()
	{
		ProfScope ps(this, CUBA_PROF_DECOMP_NUMERICAL);
		const bool flagged = p3.pcg3 && !pick.pcg2;
		Pcg3Args<T> b{};
		b.base = pcg2_args(p3, p3.cap);
		b.wFlag = p3.flags.p;
		b.pFlag = p3.flags.p + 2 * (2 * 6 * (size_t)S.numP);
		b.abortFlag = (int*)(b.pFlag + 2 * (2 * PCG3_REPL * 2 * (size_t)p3.G));
#ifdef CUBA_PCG_TIMING
		if (flagged) { CUDA_TRY(pcgTiming.alloc(8 * (size_t)p3.G)); b.timing = pcgTiming.p; }
#endif
		if (flagged) CUDA_TRY(cudaMemsetAsync(p3.flags.p, 0, sizeof(unsigned long long) * p3.flags.n, stream));
		void* args[] = { flagged ? (void*)&b : (void*)&b.base };
		CUDA_TRY(cudaLaunchCooperativeKernel(flagged ? (void*)k_pcg3<T> : (void*)k_pcg2<T>, dim3(p3.G), dim3(flagged ? PCG3_BLOCK : PCG2_BLOCK), args, p3.smem, stream));
		launches++;
		lastPcgKernel = flagged ? CUBA_PCG_KERNEL_PCG3 : CUBA_PCG_KERNEL_PCG2;
		return CUBA_OK;
	}

	// ---- k_pcg5: two-level, flag-synchronised, rows distributed over the ranks (cuba_pcg5.cuh) --------------------------
	// A launch shape of a k_pcg5 plan: k_pcg5 (256 threads, BIG or not: pcg5_legacy_shape) or the tuned one-GPU k_pcg5t
	// (cuba_pcg5t.cuh), its two-level dimensions (block_jacobi_dims: the block-Jacobi ones), kernel, block and dynamic shared
	// memory.  perSM: CTAs per SM, 0 when the plan does not fit.
	struct P5Shape {
		bool tuned = false, big = false;
		Pcg5Dims dims{}; p5t::Pcg5Dims tDims{};   // k_pcg5 / k_pcg5t
		const void* fn = nullptr; int block = PCG5_BLOCK, perSM = 0; size_t smem = 0;
	};
	// One rank's boards in 16-byte words: [2 solve halves][2 pass parities] of w, of the per-CTA partials, of the rank summaries
	// and of the coarse corrections, then the control block at 8-byte word ctl; words: 8-byte words of the whole set.
	struct P5Boards { size_t w = 0, p = 0, r = 0, c = 0, ctl = 0, words = 0; };
	// One k_pcg5 solve set up on the device (pcg5_upload): a plan's lists, coarse level and vectors, and its launch shape
	struct Pcg5Run {
		int numP = 0, G = 0, W = 1, gs = 1, apc = 1;
		P5Shape sh;
		DBuf<int> ctaRow, needPtr, needCol, local;
		DBuf<unsigned char> rowPeers;
		CoarseLevel coarse;
		DBuf<T> Linv, R0, Zhat, rcRow, rc0;
		P5Boards boards() const
		{
			const size_t NR = 3 + 6 * (size_t)(G / gs);
			P5Boards b;
			b.w = 4 * 6 * (size_t)numP; b.p = 4 * (size_t)PCG5_REPL * G * p5t::pcg5t_np(apc);
			b.r = 4 * (size_t)PCG5_REPL * W * NR; b.c = 4 * (size_t)PCG5_REPL * 6 * coarse.A;
			b.ctl = 2 * (b.w + b.p + b.r + b.c);
			b.words = b.ctl + (sizeof(Pcg5Ctl) + 7) / 8 + 2;
			return b;
		}
		Pcg5Ctl* ctl(unsigned long long* base) const { return (Pcg5Ctl*)(base + boards().ctl); }
	};
	Pcg5Run p5;                                    // the engine's own (setup_pcg5)
	DBuf<unsigned long long> p5Boards;
	P5Boards p5Layout;                             // the layout p5Boards was cleared for
	PeerMap p5Peer;                                // the peers' boards
	PcgPartition hostPP;                           // host copy of k_pcg3's row partition of the current system (setup_pcg3)
	bool p5Ok = false;
	// read by cuba_debug_get_pcg_info only: the kernel of the last solve (CUBA_PCG_KERNEL_*), counters since set_problem, and a
	// log of the cInfo flag of every k_pcg5 coarse rebuild -- rebuild n writes slot 1 + n % P5_INFO_LOG of cInfo (k_pcg4 keeps
	// slot 0), so no rebuild's outcome is overwritten by the next one and nothing is copied on the solve's path
	static constexpr int P5_INFO_LOG = 256;
	int lastPcgKernel = CUBA_PCG_KERNEL_NONE;
	long long bjRetries = 0;
	int* p5InfoSlot() const { return cInfo.p + 1 + (int)(p5.coarse.rebuilds % P5_INFO_LOG); }
	long long p5TagBound = 0;                      // conservative host-side bound on the device tag base

	// Maps one device allocation of every peer into this process (cudaIpc over NVLink peer access); the 64-byte handles travel by
	// ncclAllGather.  All ranks agree on the outcome (sum of per-rank success flags), so either everybody uses the peer path or
	// everybody keeps the NCCL one.
	int ipcExchange(void* localBase, PeerMap& m, bool& ok)
	{
		ok = false;
		if (m.mappedFor == localBase) { ok = true; return CUBA_OK; }
		m.close(rank);
		cudaIpcMemHandle_t mine;
		int good = cudaIpcGetMemHandle(&mine, localBase) == cudaSuccess ? 1 : 0;
		if (!good) cudaGetLastError();
		DBuf<char> dh;
		CUDA_TRY(dh.alloc(sizeof(cudaIpcMemHandle_t) * (size_t)world));
		CUDA_TRY(cudaMemcpyAsync(dh.p + sizeof(cudaIpcMemHandle_t) * (size_t)rank, &mine, sizeof(mine), cudaMemcpyHostToDevice, stream));
		int rc = g_nccl.AllGather(dh.p + sizeof(cudaIpcMemHandle_t) * (size_t)rank, dh.p, sizeof(cudaIpcMemHandle_t), NCCL_INT8, comm, stream);
		if (rc != 0) return fail(CUBA_ERR_COMM, "ncclAllGather (memory handles) failed");
		std::vector<cudaIpcMemHandle_t> all(world);
		CUDA_TRY(cudaMemcpyAsync(all.data(), dh.p, sizeof(cudaIpcMemHandle_t) * (size_t)world, cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		for (int r = 0; r < world && good; r++) {
			if (r == rank) { m.base[r] = localBase; continue; }
			if (cudaIpcOpenMemHandle(&m.base[r], all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); m.base[r] = nullptr; good = 0; }
		}
		// agreement
		DBuf<double> flag;
		CUDA_TRY(flag.alloc(1));
		const double mineOk = good;
		CUDA_TRY(cudaMemcpyAsync(flag.p, &mineOk, sizeof(double), cudaMemcpyHostToDevice, stream));
		rc = allreduce(flag.p, 1, false); if (rc) return rc;
		double tot = 0;
		CUDA_TRY(cudaMemcpyAsync(&tot, flag.p, sizeof(double), cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		if ((int)(tot + 0.5) != world) { m.close(rank); return CUBA_OK; }
		m.mappedFor = localBase;
		ok = true;
		return CUBA_OK;
	}

	// ---- the per-trial Hsc | bsc all-reduce over peer memory (cuba_peer_reduce.cuh) ----
	PeerMap uPeer;
	bool uPeerOk = false;
	unsigned int uEpoch = 0;
	size_t uCount = 0;             // elements of the all-reduced part of uVal
	// a buffer of the peer all-reduce holds n elements, then the signal block at this element
	static size_t peer_signal_offset(size_t n) { return (n + 1) & ~(size_t)1; }
	// the arguments of rank r of W whose buffers start at bufs[0..W-1]
	static peer::Args<T> peer_args(void* const* bufs, int r, int W, size_t n, unsigned int epoch, GridBar* bar)
	{
		peer::Args<T> a;
		const size_t sigOff = peer_signal_offset(n);
		for (int q = 0; q < peer::MAXW; q++) { a.peers[q] = nullptr; a.sigPeer[q] = nullptr; }
		for (int q = 0; q < W; q++) { a.peers[q] = (T*)bufs[q]; a.sigPeer[q] = (unsigned int*)((T*)bufs[q] + sigOff); }
		a.local = a.peers[r]; a.sigLocal = a.sigPeer[r]; a.n = n; a.rank = r; a.world = W; a.epoch = epoch; a.bar = bar;
		return a;
	}
	int launch_peer_allreduce()
	{
		peer::Args<T> pa = peer_args(uPeer.base, rank, world, uCount, ++uEpoch, gridBar);
		void* args[] = { (void*)&pa };
		CUDA_TRY(cudaLaunchCooperativeKernel((void*)peer::k_peer_allreduce<T>, dim3(numSMs), dim3(peer::BLOCK), args, 0, stream));
		launches++;
		return CUBA_OK;
	}

	int pcg5_max_agg() const { return (cfg.reserved[6] > 0 && cfg.reserved[6] < PCG5_MAXAGG) ? cfg.reserved[6] : PCG5_MAXAGG; }

	// k_pcg5's legacy (256-thread) shape for a plan: the blocks cached in shared memory, Z^ in shared memory or not, BIG or not, the
	// dynamic shared memory and the kernel -- k_pcg5, or with `ranks` k_pcg5_ranks for cuba_debug_pcg5_ranks, whose W ranks emulated
	// in one launch thus run the shape of a W-GPU run, as they run its upload, board layout and arguments.
	int pcg5_legacy_shape(const Pcg5Plan& plan, Pcg5Dims d, int W, bool ranks, P5Shape& sh)
	{
		sh = P5Shape{};
		const size_t budget = (size_t)smemMax > 4096 ? (size_t)smemMax - 2048 : 0;   // static arrays of k_pcg5: < 1 KB
		const PcgPartition& PP = plan.P;
		const size_t per = 36 * sizeof(T) + 4;
		const size_t wantCache = PP.blkMax > PCG5_REGBLK ? (size_t)(PP.blkMax - PCG5_REGBLK) : 0;
		bool big = PP.maxRows * 6 > PCG5_BLOCK;
		{
			d.capBlocks = 0; d.zhInSmem = 0;
			const size_t base = Pcg5Layout<T>(d).total + 64;
			if (base > budget) return CUBA_OK;
			const size_t zhBytes = (size_t)d.needMax * 36 * sizeof(T);
			size_t used = base + wantCache * per;
			if (used + zhBytes <= budget) { d.zhInSmem = 1; used += zhBytes; }
			const size_t fixed = used - wantCache * per;
			d.capBlocks = (int)std::min(wantCache, (budget - fixed) / per);
			// blocks would have to be streamed from the global copy every pass: the variant without register-resident blocks streams
			// with eighteen 16-byte loads in flight per thread (the register variant can afford six 8-byte loads)
			if ((size_t)d.capBlocks < wantCache) big = true;
			if (big) d.capBlocks = (int)std::min((size_t)PP.blkMax, (budget - fixed) / per);
		}
		const size_t smem = std::max(Pcg5Layout<T>(d).total, Pcg5Layout<T>(block_jacobi_dims(d, plan.G, W)).total);
		if (smem > (size_t)smemMax - 1024) return CUBA_OK;
		const void* fn = ranks ? (big ? (const void*)k_pcg5_ranks<T, true> : (const void*)k_pcg5_ranks<T, false>)
		                       : (big ? (const void*)k_pcg5<T, true> : (const void*)k_pcg5<T, false>);
		CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
		int perSM = 0;
		CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, fn, PCG5_BLOCK, smem));
		sh.dims = d; sh.smem = smem; sh.big = big; sh.fn = fn; sh.perSM = perSM;
		return CUBA_OK;
	}

	// Partition of the rows over world x G virtual CTAs, aggregates aligned with the ranks, shared-memory budget, boards.
	int setup_pcg5()
	{
		const int numP = S.numP, W = pick.dist ? world : 1;
		const size_t budget = (size_t)smemMax > 4096 ? (size_t)smemMax - 2048 : 0;   // static arrays of k_pcg5: < 1 KB
		// rows over world x G virtual CTAs (about eight rows each, never more than 42: one thread per (row, component) pair in the
		// row sums), rank-aligned aggregates, halo masks: cuba_structure.cpp (CPU-tested through cuba_debug_pcg5_plan)
		const int maxAgg = pcg5_max_agg();
		// the tuned shape (cuba_pcg5t.cuh): a solve on one GPU whose blocks fit registers + shared memory, with apc aggregates per
		// CTA -- the largest apc <= p5t::DEFAULT_APC (CUBA_PCG5_AGGS_PER_CTA: another bound, 1 = one aggregate per CTA group as
		// k_pcg5) whose plan exists and whose shared memory fits; every other shape: one aggregate per group of gs CTAs
		const bool tryTuned = W == 1 && !getenv("CUBA_PCG5_LEGACY");
		int apcTop = p5t::DEFAULT_APC;
		if (const char* e = getenv("CUBA_PCG5_AGGS_PER_CTA")) apcTop = std::min(3, std::max(1, atoi(e)));
		Pcg5Plan plan;
		P5Shape sh;
		for (int apc = tryTuned ? apcTop : 1; apc >= 1 && !sh.tuned; apc--) {
			build_pcg5_plan(numP, S.nfull, S.fRowPtr, S.fColInd, W, numSMs, maxAgg, 2 * PCG5_BLOCK / 6, plan, &hostPP, apc);
			if (!plan.ok) continue;
			if (!tryTuned) break;
			using TS = p5t::Pcg5Shape;
			p5t::Pcg5Dims t = pcg5t_plan_dims(plan);
			if (plan.P.maxRows * 6 <= TS::BLOCK && p5t::pcg5t_fit<T>(t, plan.P.blkMax, apc, budget)) {
				const size_t smemT = std::max(p5t::Pcg5Layout<T>(t).total, p5t::Pcg5Layout<T>(block_jacobi_dims(t, plan.G, W)).total);
				const void* fn = apc == 3 ? (const void*)p5t::k_pcg5t<T, 3> : apc == 2 ? (const void*)p5t::k_pcg5t<T, 2> : (const void*)p5t::k_pcg5t<T, 1>;
				int perSM = 0;
				if (smemT <= (size_t)smemMax - 1024 && cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemT) == cudaSuccess &&
					cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, fn, TS::BLOCK, smemT) == cudaSuccess && perSM >= 1) {
					sh.tuned = true; sh.tDims = t; sh.fn = fn; sh.block = TS::BLOCK; sh.smem = smemT; sh.perSM = perSM;
				} else cudaGetLastError();
			}
			// the other shapes take one aggregate per CTA group
			if (!sh.tuned && apc == 1) break;
		}
		if (!plan.ok) return CUBA_OK;
		if (!sh.tuned) {
			int rc = pcg5_legacy_shape(plan, pcg5_plan_dims(plan, W), W, false, sh); if (rc) return rc;
			if (sh.perSM < 1) return CUBA_OK;
		}
		auto show = [&](const auto& d) {
			fprintf(stderr, "pcg5: world %d G %d gs %d A %d aggsPerCta %d needMax %d maxRows %d blkMax %d maxNeedAgg %d zhInSmem %d sliceRows %d cap %d smem %zu\n",
				W, plan.G, plan.gs, plan.A, plan.apc, d.needMax, d.maxRows, plan.P.blkMax, d.maxNeedAgg, d.zhInSmem, d.sliceRows, d.capBlocks, sh.smem);
			fprintf(stderr, "pcg5: shape %s, %d threads\n", sh.big ? "big" : sh.tuned ? "tuned" : "legacy", sh.block);
		};
		if (getenv("CUBA_PCG_VERBOSE")) { if (sh.tuned) show(sh.tDims); else show(sh.dims); }
		int rc = pcg5_upload(p5, plan, sh, W, &arena); if (rc) return rc;
		CUDA_TRY(cZx.alloc(36 * (size_t)numP)); CUDA_TRY(cU.alloc(36 * (size_t)S.nfull)); CUDA_TRY(cInfo.alloc(1 + P5_INFO_LOG));
		CUDA_TRY(cudaMemsetAsync(cInfo.p, 0, sizeof(int) * cInfo.n, stream));
		CUDA_TRY(fHat.alloc(36 * (size_t)S.nfull));
		if (coarse_kernel(plan.A) == CUBA_COARSE_KERNEL_DENSE) CUDA_TRY(cdT.alloc(cdense::scratch_doubles(plan.A)));
		const P5Boards b = p5.boards();
		const bool fresh = !p5Boards.p || b.words > p5Boards.cap || b.w != p5Layout.w || b.p != p5Layout.p || b.r != p5Layout.r || b.c != p5Layout.c;
		if (fresh) {
			// the tag protocol needs boards that start out as zeros; a layout change invalidates every mapping and every tag
			if (p5Peer.mappedFor) { CUDA_TRY(cudaStreamSynchronize(stream)); p5Peer.close(rank); }
			CUDA_TRY(p5Boards.alloc(std::max(b.words, (size_t)(1u << 18))));
			CUDA_TRY(cudaMemsetAsync(p5Boards.p, 0, sizeof(unsigned long long) * p5Boards.cap, stream));
			p5Layout = b;
			p5TagBound = 0;
		}
		if (W > 1) {
			bool ok = false;
			rc = ipcExchange((void*)p5Boards.p, p5Peer, ok); if (rc) return rc;
			if (!ok) {
				if (rank == 0) fprintf(stderr, "cuba_b200: cudaIpc mapping of the peers' PCG boards failed; keeping the replicated PCG\n");
				return CUBA_OK;
			}
		} else p5Peer.base[rank] = (void*)p5Boards.p;
		p5Ok = true;
		return CUBA_OK;
	}

	// R for a solve of `plan` over W ranks in shape sh: the plan's lists and coarse level (through the pinned arena when one is
	// given), the vectors of the preparation
	int pcg5_upload(Pcg5Run& R, const Pcg5Plan& plan, const P5Shape& sh, int W, PinnedArena* arena)
	{
		R.numP = S.numP; R.G = plan.G; R.W = W; R.gs = plan.gs; R.apc = plan.apc; R.sh = sh;
		const PcgPartition& PP = plan.P;
		CUDA_TRY(R.ctaRow.upload(PP.rows, stream, arena)); CUDA_TRY(R.needPtr.upload(PP.nptr, stream, arena)); CUDA_TRY(R.needCol.upload(PP.ncol, stream, arena));
		CUDA_TRY(R.local.upload(PP.local, stream, arena)); CUDA_TRY(R.rowPeers.upload(plan.rowPeers, stream, arena));
		int rc = R.coarse.upload(plan.C, stream, arena); if (rc) return rc;
		const size_t nP = (size_t)S.numP;
		CUDA_TRY(R.Linv.alloc(36 * nP)); CUDA_TRY(R.R0.alloc(6 * nP)); CUDA_TRY(R.Zhat.alloc(36 * nP)); CUDA_TRY(R.rcRow.alloc(6 * nP));
		CUDA_TRY(R.rc0.alloc(std::max(6 * plan.A, 1)));
		return CUBA_OK;
	}

	// blocked symmetric sweep on the whole chip (cuba_coarse.cuh): one persistent cooperative kernel; tiles holds
	// cdense::scratch_doubles(A) doubles, bar a zeroed or reused GridBar
	int launch_coarse_dense(const double* AcP, int A, double* tiles, float* AcInv, int* info, GridBar* bar)
	{
		CUDA_TRY(cudaFuncSetAttribute(cdense::k_coarse_dense, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cdense::SMEM));
		cdense::Args da;
		da.AcP = AcP; da.A = A; da.T = tiles; da.AcInv = AcInv; da.info = info; da.bar = bar;
		void* dargs[] = { (void*)&da };
		CUDA_TRY(cudaLaunchCooperativeKernel((void*)cdense::k_coarse_dense, dim3(numSMs), dim3(cdense::WARPS * 32), dargs, cdense::SMEM, stream));
		launches++;
		return CUBA_OK;
	}

	// scratch of a coarse rebuild: the coarse basis Zx of the current state, U [36 nfull], and for k_coarse_dense its tiles and a
	// zeroed or reused GridBar
	struct CoarseScratch { T* Zx; double* U; double* tiles; GridBar* bar; };
	CoarseScratch coarse_scratch() const { return { cZx.p, cU.p, cdT.p, gridBar.p }; }

	// coarse matrix Ac = Z^T S Z of the current system and its inverse (fp32), for the aggregates of L; info: 0 inverted, 1 not
	// positive definite (AcInv zeroed).  The inverse: coarse_kernel(A).
	int launch_coarse_setup(const CoarseLevel& L, const CoarseScratch& s, int* info)
	{
		const int A = L.A, nblkP = A * (A + 1) / 2;
		KLAUNCH(k_coarse_project<T>, 36LL * S.nfull, fVal.p, L.rowOf.p, fColInd.p, S.nfull, s.Zx, s.U);
		KLAUNCH(k_coarse_assemble, (long long)nblkP * 36, L.cbPtr.p, L.cbList.p, s.U, nblkP, L.AcP.p);
		if (coarse_kernel(A) == CUBA_COARSE_KERNEL_DENSE) return launch_coarse_dense(L.AcP, A, s.tiles, L.AcInv, info, s.bar);
		k_coarse_invert<T><<<1, 1024, coarse_invert_smem(A), stream>>>(L.AcP, A, L.AcInv, info);
		launches++;
		CUDA_TRY(cudaGetLastError());
		return CUBA_OK;
	}

	// The coarse matrix Ac = Z^T S Z and its inverse are rebuilt only now and then: ANY symmetric positive definite stand-in for
	// Ac^-1 keeps M^-1 = D^-1 + Z B Z^T a valid preconditioner, and the coarse operator of an earlier damping / linearisation
	// preconditions as well as the current one (CPU prototype: 26..201 iterations over ten LM iterations with a fresh inverse,
	// 26..193 with one that is refreshed every fifth iteration).
	// Measured limits of that freedom: a coarse inverse from an 81x larger damping costs nothing, one from a 1e5x larger damping
	// costs 8x the iterations (1 276 vs 149 on kitti00_shaped) -> it is also rebuilt when the damping moved by more than 300x.
	bool coarse_due(const CoarseLevel& L) const
	{
		const int refreshEvery = cfg.reserved[4] > 0 ? cfg.reserved[4] : 8;
		const double lamRatio = (L.valid && L.lambda > 0 && curLambda > 0) ? std::max(curLambda / L.lambda, L.lambda / curLambda) : 1.0;
		return !L.valid || L.age >= refreshEvery || lamRatio > 300.0;
	}
	// before a two-level solve: L rebuilt when due, then the solve counted
	int coarse_refresh(CoarseLevel& L, const CoarseScratch& s, int* info)
	{
		if (coarse_due(L)) {
			int rc = launch_coarse_setup(L, s, info); if (rc) return rc;
			L.valid = true; L.age = 0; L.lambda = curLambda; L.rebuilds++;
		}
		L.age++;
		return CUBA_OK;
	}

	// nothing an earlier solve left behind is reused: block-Jacobi first, both coarse inverses rebuilt at their next two-level solve
	void forget_solves() { tlActive = false; p4.coarse.forget(); p5.coarse.forget(); }

	// The preparation of a solve of R on the current system: k_pcg5_prep_rows for each of the n control blocks ctl[] (the rows of
	// Linv, R0, Z^ and rc0 are the same on every rank: computed once, each rank's breakdown counter counted in its own control
	// block) and, two-level, the coarse basis, rc0 and the coarse level (coarse_refresh).
	int pcg5_prepare(Pcg5Run& R, bool twoLevel, Pcg5Ctl* const* ctl, int n, const CoarseScratch& s, int* info)
	{
		const int numP = R.numP, A = twoLevel ? R.coarse.A : 0;
		if (twoLevel) KLAUNCH(k_coarse_basis<T>, numP, pose[cur].p, numP, s.Zx);
		Pcg5PrepArgs<T> pa;
		pa.fRowPtr = fRowPtr; pa.fColInd = fColInd; pa.fVal = fVal; pa.b = bsc; pa.Zx = s.Zx; pa.numP = numP; pa.A = A; pa.aggRow = R.coarse.aggRow;
		pa.zhatFp32 = R.sh.tuned ? 1 : 0;
		pa.Linv = R.Linv; pa.R0 = R.R0; pa.Zhat = R.Zhat; pa.rcRow = R.rcRow; pa.rc0 = R.rc0;
		for (int r = 0; r < n; r++) {
			pa.ctl = ctl[r];
			k_pcg5_prep_rows<T><<<(numP + 127) / 128, 128, 0, stream>>>(pa);
			launches++;
		}
		if (twoLevel) {
			k_pcg5_prep_rc<T><<<(6 * A + 127) / 128, 128, 0, stream>>>(pa);
			launches++;
			int rc = coarse_refresh(R.coarse, s, info); if (rc) return rc;
		}
		CUDA_TRY(cudaGetLastError());
		return CUBA_OK;
	}

	// The arguments of R's solve for its rank r of W: rank q's boards at bases[q] (bases[r]: this rank's own), A^ into hat, x and
	// status as given.  k_pcg5 (Pcg5Args) and k_pcg5t (p5t::Pcg5Args) differ only in their dims and k_pcg5t's aggRow.
	template <typename Args>
	void pcg5_args(Args& a, const Pcg5Run& R, bool twoLevel, int r, int W, unsigned long long* const* bases, T* hat, T* x, PcgStatus* status) const
	{
		const P5Boards b = R.boards();
		a.fRowPtr = fRowPtr; a.fColInd = fColInd; a.fLocal = R.local; a.fVal = fVal; a.fHat = hat;
		a.ctaRow = R.ctaRow; a.needPtr = R.needPtr; a.needCol = R.needCol;
		a.numP = R.numP; a.G = R.G; a.rank = r; a.world = W;
		a.Linv = R.Linv; a.R0 = R.R0; a.Zhat = R.Zhat; a.rc0 = R.rc0; a.x = x;
		a.maxIters = pcg_max_iters(); a.tol2 = pcg_tol2();
		a.status = status;
		a.AcInv = R.coarse.AcInv; a.naPtr = R.coarse.naPtr; a.naList = R.coarse.naList; a.needAgg = R.coarse.needAgg;
		a.A = twoLevel ? R.coarse.A : 0; a.gs = R.gs;
		for (int q = 0; q < PCG5_MAXWORLD; q++) { a.peerW[q] = nullptr; a.peerR[q] = nullptr; a.peerCtl[q] = nullptr; }
		for (int q = 0; q < W; q++) { a.peerW[q] = bases[q]; a.peerR[q] = bases[q] + 2 * (b.w + b.p); a.peerCtl[q] = (Pcg5Ctl*)(bases[q] + b.ctl); }
		unsigned long long* own = bases[r];
		a.wBoard = own; a.pBoard = own + 2 * b.w; a.rBoard = own + 2 * (b.w + b.p); a.cBoard = own + 2 * (b.w + b.p + b.r);
		a.rowPeers = R.rowPeers; a.ctl = (Pcg5Ctl*)(own + b.ctl);
		a.timing = nullptr;
		if constexpr (std::is_same<Args, Pcg5Args<T>>::value) a.dims = R.sh.dims;
		else { a.dims = R.sh.tDims; a.aggRow = R.coarse.aggRow; }
		if (!twoLevel) a.dims = block_jacobi_dims(a.dims, R.G, R.W);
	}

	int launch_pcg5(bool twoLevel)
	{
		ProfScope ps(this, CUBA_PROF_DECOMP_NUMERICAL);
		const int maxIters = pcg_max_iters();
		// tags are 32 bits: long before the device tag base can wrap, every rank (same arithmetic everywhere) clears its boards
		p5TagBound += (long long)maxIters + 8;
		if (p5TagBound > (1LL << 31)) {
			if (pick.dist) { int rc0 = allreduce(&dScal.p->v[7], 1, false); if (rc0) return rc0; }   // nobody still writes into a peer's boards
			CUDA_TRY(cudaMemsetAsync(p5Boards.p, 0, sizeof(unsigned long long) * p5Boards.cap, stream));
			if (pick.dist) { int rc0 = allreduce(&dScal.p->v[7], 1, false); if (rc0) return rc0; }
			p5TagBound = (long long)maxIters + 8;
		}
		Pcg5Ctl* ctl = p5.ctl(p5Boards.p);
		int rc = pcg5_prepare(p5, twoLevel, &ctl, 1, coarse_scratch(), p5InfoSlot()); if (rc) return rc;
#ifdef CUBA_PCG_TIMING
		CUDA_TRY(pcgTiming.alloc(8 * (size_t)p5.G));
#endif
		if (pick.dist) CUDA_TRY(cudaMemsetAsync(xp.p, 0, sizeof(T) * 6 * (size_t)S.numP, stream));     // rows of the other ranks: summed in below
		// a replicated solve (p5.W == 1, also on a multi-rank engine) is rank 0 of one, on this rank's own boards
		unsigned long long* bases[PCG5_MAXWORLD];
		for (int r = 0; r < p5.W; r++) bases[r] = (unsigned long long*)p5Peer.base[pick.dist ? r : rank];
		auto launch = [&](auto& a) {
			pcg5_args(a, p5, twoLevel, pick.dist ? rank : 0, p5.W, bases, fHat.p, xp.p, &dScal.p->pcg);
#ifdef CUBA_PCG_TIMING
			a.timing = pcgTiming.p;
#endif
			void* args[] = { (void*)&a };
			return cudaLaunchCooperativeKernel(p5.sh.fn, dim3(p5.G), dim3(p5.sh.block), args, p5.sh.smem, stream);
		};
		Pcg5Args<T> a;
		p5t::Pcg5Args<T> at;
		CUDA_TRY(p5.sh.tuned ? launch(at) : launch(a));
		k_pcg5_commit<<<1, 1, 0, stream>>>(ctl);
		launches += 2;
		CUDA_TRY(cudaGetLastError());
		if (pick.dist) { rc = allreduce(xp.p, 6 * (size_t)S.numP, true); if (rc) return rc; }
		lastPcgTwoLevel = twoLevel;
		lastPcgKernel = p5.sh.tuned ? CUBA_PCG_KERNEL_PCG5T : p5.sh.big ? CUBA_PCG_KERNEL_PCG5_BIG : CUBA_PCG_KERNEL_PCG5;
		return CUBA_OK;
	}

	// ---- the direct solver (cuba_dense_chol.cuh) ---------------------------------------------------------------------------
	bool denseSolve = false;        // the structure was built for the direct solver (set_problem, from linSolver)
	DBuf<int> dcMap;                // packed lower block triangle -> block of the full BSR (build_dense_block_map)
	DBuf<double> dcTiles, dcY;
	// CTAs of k_dense_chol for an n x n system: enough for the widest phase (the first trailing update), at most one per SM
	int dense_grid(int n) const
	{
		const long long nt = dchol::tile_rows(n), widest = std::max(nt * (nt - 1) / 2, nt);
		return (int)std::max(1LL, std::min<long long>(numSMs, (widest + dchol::WARPS - 1) / dchol::WARPS));
	}
	void release_dense() { dcMap.release(); dcTiles.release(); dcY.release(); }
	int setup_dense()
	{
		const int n = 6 * S.numP;
		std::vector<int> map;
		build_dense_block_map(S.numP, S.fRowPtr, S.fColInd, map);
		CUDA_TRY(dcMap.upload(map, stream));
		CUDA_TRY(dcTiles.alloc(dchol::tile_doubles(n))); CUDA_TRY(dcY.alloc(dchol::rhs_doubles(n)));
		return CUBA_OK;
	}
	template <typename U>
	int launch_dense_chol(const dchol::Args<U>& a)
	{
		CUDA_TRY(cudaFuncSetAttribute(dchol::k_dense_chol<U>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dchol::SMEM));
		void* args[] = { (void*)&a };
		CUDA_TRY(cudaLaunchCooperativeKernel((void*)dchol::k_dense_chol<U>, dim3(dense_grid(a.n)), dim3(dchol::WARPS * 32), args, dchol::SMEM, stream));
		launches++;
		return CUBA_OK;
	}
	// S xp = bsc by Cholesky: status slot iters 0, status 0 (2: S not positive definite, xp = 0)
	int launch_dense()
	{
		if (!dcTiles.p) return fail(CUBA_ERR_STATE, "dense solve: the problem has no reduced camera system (no free pose or no free landmark)");
		ProfScope ps(this, CUBA_PROF_DECOMP_NUMERICAL);
		dchol::Args<T> a;
		a.fVal = fVal; a.blkMap = dcMap; a.dense = nullptr; a.b = bsc; a.n = 6 * S.numP;
		a.tl = dcTiles; a.y = dcY; a.x = xp; a.status = &dScal.p->pcg; a.info = nullptr; a.bar = gridBar;
		const int rc = launch_dense_chol(a); if (rc) return rc;
		lastPcgTwoLevel = false;
		lastPcgKernel = CUBA_PCG_KERNEL_DENSE;
		return CUBA_OK;
	}

	// the reduced-system solve of the structure's solver
	int launch_solver() { return denseSolve ? launch_dense() : launch_pcg(); }

	int launch_pcg()
	{
		lastPcgTwoLevel = false;
		const PcgStep& s = forceBlockJacobi ? pick.retry : tlActive ? pick.later : pick.first;
		if (s.p5 && p5Ok) return launch_pcg5(s.twoLevel);
		if (s.p4 && p4.ok) return launch_pcg4();
		return launch_pcg3();
	}

	int launch_backsub(T lambda)
	{
		ProfScope ps(this, CUBA_PROF_SCHUR_COMPLEMENT);
		if (ntiles > 0 && S.numL > 0) return stages.mixed ? launch_backsub(HplF.p, lambda) : launch_backsub(Hpl.p, lambda);
		return CUBA_OK;
	}
	// k_backsub on Hpl blocks of type HT: T, or float under mixed precision
	template <typename HT>
	int launch_backsub(const HT* hpl, T lambda)
	{
		BacksubArgs<T, HT> a;
		a.Hpl = hpl; a.invHll = invHll; a.bl = bl; a.xp = xp; a.ip = e_ip; a.hpl = e_hpl; a.lmPtr = tilePtr; a.tileLm = tileLm;
		a.numL = S.numL; a.lambda = lambda; a.XwCur = Xw[cur]; a.XwTrial = Xw[cur ^ 1]; a.xl = xl; a.scalePartial = scalePartialL;
		if (stages.tileSize == 128) k_backsub<T, 128, HT><<<ntiles, 128, 0, stream>>>(a);
		else k_backsub<T, 256, HT><<<ntiles, 256, 0, stream>>>(a);
		launches++;
		CUDA_TRY(cudaGetLastError());
		return CUBA_OK;
	}

	// Schur + PCG + back-substitution.  Leaves xp/xl, the trial landmarks and the landmark scale partials.
	int stage_solve(double lambda, int* iters, int* ok) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "solve before set_problem");
		const T lam = (T)lambda;
		curLambda = lambda;
		int rc = launch_schur(lam); if (rc) return rc;
		int nScaleL = 0;
		if (S.numP > 0 && S.numL > 0) {
			rc = launch_solver(); if (rc) return rc;
			rc = launch_backsub(lam); if (rc) return rc;
			nScaleL = ntiles;
		} else if (S.numP > 0) {
			k_solve_poses_only<T><<<(S.numP + 127) / 128, 128, 0, stream>>>(Hpp, bp, S.numP, lam, xp);
			launches++;
			CUDA_TRY(cudaGetLastError());
			hScal->pcg.iters = 0; hScal->pcg.status = 0;
			lastPcgKernel = CUBA_PCG_KERNEL_NONE;
		} else if (S.numL > 0) {
			nScaleL = (S.numL + RED_BLOCK - 1) / RED_BLOCK;
			k_solve_landmarks_only<T><<<nScaleL, RED_BLOCK, 0, stream>>>(invHll, bl, S.numL, lam, Xw[cur], Xw[cur ^ 1], xl, scalePartialL);
			launches++;
			CUDA_TRY(cudaGetLastError());
		}
		nScaleLandmark = nScaleL;
		solvedLambda = lambda;
		if (iters || ok) {
			rc = fetchScalars(); if (rc) return rc;
			const bool usedPcg = S.numP > 0 && S.numL > 0;
			if (usedPcg) note_pcg_iters(hScal->pcg.iters);
			if (iters) *iters = usedPcg ? hScal->pcg.iters : 0;
			if (ok) *ok = usedPcg ? (hScal->pcg.status == 0) : 1;
		}
		return CUBA_OK;
	}
	int nScaleLandmark = 0;
	double solvedLambda = 0;

	// pose update + trial chi2 + scale; results in dScal->v[1] (chi2), v[2..3] (scale parts)
	int stage_update(double lambda, double* chi, double* scale) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "update before set_problem");
		const T lam = (T)lambda;
		{
			ProfScope ps(this, CUBA_PROF_UPDATE);
			if (S.numP > 0) {
				k_update_poses<T><<<nPoseBlocks, RED_BLOCK, 0, stream>>>(xp, bp, S.numP, lam, pose[cur], pose[cur ^ 1], scalePartialP);
				launches++;
				CUDA_TRY(cudaGetLastError());
			}
		}
		int rc = launch_chi2(cur ^ 1, 1, false); if (rc) return rc;
		// scale = sum over [xp;xl] of x (lambda x + b): pose part is replicated, landmark part is sharded
		rc = launch_sum(scalePartialL, nScaleLandmark, scalePartialP, S.numP > 0 ? nPoseBlocks : 0, nullptr, 0, 2); if (rc) return rc;
		if (world > 1) { rc = allreduce(&dScal.p->v[1], 2, false); if (rc) return rc; }   // trial chi2 and the landmark part of the scale: adjacent slots
		rc = fetchScalars(); if (rc) return rc;
		trialValid = true;
		if (chi) *chi = hScal->v[1];
		if (scale) *scale = hScal->v[2] + hScal->v[3];
		return CUBA_OK;
	}

	int stage_commit(int accept) override
	{
		if (!trialValid) return fail(CUBA_ERR_STATE, "commit without a trial state");
		if (accept) cur ^= 1;
		trialValid = false;
		return CUBA_OK;
	}

	// ---- the LM loop: reference src/cuda_bundle_adjustment.cpp:793-857 ---------------------------------
	int optimize(int niter, cuba_iter_stat* stats, int* nstats) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "optimize before set_problem");
		if (lvOn && lvIncluded == 0) { if (nstats) *nstats = 0; return CUBA_OK; }   // every edge at level 1: nothing to optimise
		double nu = 2, lambda = 0, F = 0;
		int n = 0;
		forget_solves(); forceBlockJacobi = false;     // results never depend on what the engine solved before
		bool haveF = false;
		for (int it = 0; it < niter; it++) {
			double chi0 = 0;
			int rc = stage_linearize(&chi0); if (rc) return rc;
			// after an accepted trial the reference recomputes the same residuals (cpp:808); the value is F
			if (!haveF) F = chi0;
			F = chi0; haveF = true;
			if (it == 0) {
				double md = 0;
				rc = stage_max_diagonal(&md); if (rc) return rc;
				lambda = lm::initial_lambda(md);
			}
			int q = 0, trials = 0, pcgIters = 0, pcgFailed = 0;
			double rho = -1;
			for (; q < lm::MAX_TRIALS && rho < 0; q++) {
				trials++;
				int iters = 0, ok = 1;
				double Fhat = 0, scale = 0;
				for (int attempt = 0; attempt < 2; attempt++) {
					rc = stage_solve(lambda, nullptr, nullptr); if (rc) return rc;
					rc = stage_update(lambda, &Fhat, &scale); if (rc) return rc;
					if (!(S.numP > 0 && S.numL > 0)) break;
					const PcgStatus& ps = hScal->pcg;
					iters += ps.iters;
					if (ps.status == 3) return fail(CUBA_ERR_COMM, "PCG: a CTA or a peer GPU stopped answering (flag exchange timed out)");
					// The reference's direct solve fails only when the factorisation does (cuda_linear_solver.cpp:406-410).  Here: a solve
					// that ran into the iteration cap is still used when its residual fell far enough for an LM step; a breakdown of a
					// two-level solve (the fp32 coarse inverse lost definiteness) is retried once with block-Jacobi alone.
					const double loose = sizeof(T) == 8 ? 1e-6 : 1e-3;
					ok = ps.status == 0 || (ps.status == 1 && ps.rz0 > 0 && ps.rz <= loose * loose * ps.rz0);
					if (ps.status == 2 && lastPcgTwoLevel && attempt == 0) {
						forceBlockJacobi = true; p4.coarse.valid = false; p5.coarse.valid = false; bjRetries++;
						rc = stage_commit(0); if (rc) return rc;
						continue;
					}
					break;
				}
				forceBlockJacobi = false;
				if (S.numP > 0 && S.numL > 0) note_pcg_iters(hScal->pcg.iters);
				pcgIters += iters; if (!ok) pcgFailed++;
				rho = ok ? lm::gain_ratio(F, Fhat, scale) : -1;
				if (lm::update_damping(rho, lambda, nu)) {
					F = Fhat;
					rc = stage_commit(1); if (rc) return rc;
					break;
				}
				rc = stage_commit(0); if (rc) return rc;
			}
			if (stats) {
				stats[n].iteration = it; stats[n].trials = trials; stats[n].chi2 = F; stats[n].lambda = lambda;
				stats[n].pcg_iters = pcgIters; stats[n].pcg_failed = pcgFailed;
			}
			n++;
			if (lm::stop(q, rho, lambda)) break;
		}
		if (nstats) *nstats = n;
		resolveProfile();   // the stream is idle (every trial ends with a fetch): recycle the profile events instead of hoarding them
		return CUBA_OK;
	}

	// The landmarks get_state returns: Xw[cur], or in landmark-sharded runs every rank's own range all-gathered into the trial
	// buffer, which is free between LM iterations.  (!comm: a CUBA_DRY_SHARD engine returns its own buffer -- its landmarks updated,
	// the others as uploaded.)
	int gather_landmarks(const T*& xw)
	{
		xw = Xw[cur].p;
		if (!(world > 1 && comm && S.numL > 0)) return CUBA_OK;
		// all-gather of the sharded landmarks: every rank broadcasts its own range in place (one grouped NCCL call)
		T* tmp = Xw[cur ^ 1].p;
		trialValid = false;
		CUDA_TRY(cudaMemcpyAsync(tmp, Xw[cur].p, sizeof(T) * 4 * (size_t)S.Lall, cudaMemcpyDeviceToDevice, stream));
		if (shardBoundValid) {
			const int dt = sizeof(T) == 8 ? NCCL_FLOAT64 : NCCL_FLOAT32;
			g_nccl.GroupStart();
			int rcn = 0;
			for (int r = 0; r < world; r++) {
				const int b0 = std::min(shardBound[r], S.numL), b1 = std::min(shardBound[r + 1], S.numL);     // fixed landmarks never change
				if (b1 > b0) rcn |= g_nccl.Broadcast(tmp + 4 * (size_t)b0, tmp + 4 * (size_t)b0, 4 * (size_t)(b1 - b0), dt, r, comm, stream);
			}
			rcn |= g_nccl.GroupEnd();
			if (rcn != 0) return fail(CUBA_ERR_COMM, "ncclBroadcast (landmark gather) failed");
		} else {
			// host-built structure (debug path): zero the foreign entries, sum over ranks
			CUDA_TRY(cudaMemsetAsync(tmp, 0, sizeof(T) * 4 * (size_t)S.Lall, stream));
			if (S.lmEnd > S.lmBeg)
				CUDA_TRY(cudaMemcpyAsync(tmp + 4 * (size_t)S.lmBeg, Xw[cur].p + 4 * (size_t)S.lmBeg, sizeof(T) * 4 * (size_t)(S.lmEnd - S.lmBeg), cudaMemcpyDeviceToDevice, stream));
			int rc = allreduce(tmp, 4 * (size_t)S.Lall, true); if (rc) return rc;
		}
		xw = tmp;
		return CUBA_OK;
	}

	int get_state(double* q, double* t, double* X) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "get_state before set_problem");
		std::vector<T> hp((size_t)S.Pall * 8), hx((size_t)S.Lall * 4);
		g_d2hBytes += (long long)(sizeof(T) * (hp.size() + hx.size()));
		CUDA_TRY(cudaMemcpyAsync(hp.data(), pose[cur].p, sizeof(T) * hp.size(), cudaMemcpyDeviceToHost, stream));
		const T* xw = nullptr;
		int rc = gather_landmarks(xw); if (rc) return rc;
		CUDA_TRY(cudaMemcpyAsync(hx.data(), xw, sizeof(T) * hx.size(), cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		for (int i = 0; i < S.Pall; i++) {
			if (q) for (int k = 0; k < 4; k++) q[4 * (size_t)i + k] = (double)hp[8 * (size_t)i + k];
			if (t) for (int k = 0; k < 3; k++) t[3 * (size_t)i + k] = (double)hp[8 * (size_t)i + 4 + k];
		}
		if (X) for (int i = 0; i < S.Lall; i++) for (int k = 0; k < 3; k++) X[3 * (size_t)i + k] = (double)hx[4 * (size_t)i + k];
		return CUBA_OK;
	}
	int get_state_device(double* q, double* t, double* X, cudaStream_t caller) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "get_state before set_problem");
		return on_caller_stream(caller, [&] {
			const T* xw = nullptr;
			int rc = gather_landmarks(xw); if (rc) return rc;
			KLAUNCH(pio::k_unpack_state<T>, std::max(S.Pall, S.Lall), pose[cur].p, xw, S.Pall, S.Lall, q, t, X);
			return CUBA_OK;
		});
	}

	// per-edge chi2 into out[E] on the device (chiSq, or the caller's array), summed over the ranks of a landmark-sharded run
	int chi_sqs_into(double* out)
	{
		if (S.E > 0) CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(double) * (size_t)S.E, stream));
		if (S.eLocal > 0) {
			ChiArgs<T> a = chiArgs(cur);
			if (lvOn) a.om = e_om0;      // edges at level 1 report omega |r|^2 with the caller's omega
			k_chi_sqs<T><<<(S.eLocal + 255) / 256, 256, 0, stream>>>(a, e_user, out);
			launches++;
			CUDA_TRY(cudaGetLastError());
		}
		if (world > 1) { int rc = allreduce(out, (size_t)S.E, false); if (rc) return rc; }
		return CUBA_OK;
	}
	int get_chi2(double* out) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "get_chi2 before set_problem");
		int rc = chi_sqs_into(chiSq.p); if (rc) return rc;
		g_d2hBytes += (long long)(sizeof(double) * (size_t)S.E);
		CUDA_TRY(cudaMemcpyAsync(out, chiSq.p, sizeof(double) * (size_t)S.E, cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		return CUBA_OK;
	}
	int get_chi2_device(double* out, cudaStream_t caller) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "get_chi2 before set_problem");
		return on_caller_stream(caller, [&] { return chi_sqs_into(out); });
	}

	// ---- edge levels (cuba_levels.cuh) ----------------------------------------------------------------
	// first level call after a set_problem: keep the unmasked omega, every level 0
	int levels_init()
	{
		if (lvOn) return CUBA_OK;
		const int eL = S.eLocal;
		CUDA_TRY(e_om0.alloc(eL));
		if (eL > 0) CUDA_TRY(cudaMemcpyAsync(e_om0.p, e_om.p, sizeof(T) * (size_t)eL, cudaMemcpyDeviceToDevice, stream));
		CUDA_TRY(lvLevel.alloc((size_t)std::max(S.E, 1)));
		CUDA_TRY(cudaMemsetAsync(lvLevel.p, 0, (size_t)std::max(S.E, 1), stream));
		// the pose-major source list: the device builder keeps it, the host builder has it in S only
		if (cfg.reserved[1] == 1) CUDA_TRY(g_psrc.upload(S.p_src, stream));
		lvOn = true;
		lvIncluded = S.E;
		return CUBA_OK;
	}
	// the mask into the three omega streams; the same streams as a set_problem whose omega is 0 on the edges at level 1
	int levels_scatter()
	{
		const int eL = S.eLocal;
		KLAUNCH(lv::k_mask_omega<T>, eL, e_om0.p, e_user.p, lvLevel.p, eL, e_om.p);
		KLAUNCH(lv::k_pose_omega<T>, eL, g_psrc.p, posePtr.p, S.numP, eL, e_om.p, p_om.p);
		int rc = jh4_emit(); if (rc) return rc;
		// the system changed: nothing an earlier solve left behind may be reused (as after refresh_values; the estimate stays)
		trialValid = false;
		forget_solves();
		return CUBA_OK;
	}
	int set_edge_levels(const uint8_t* levels) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "set_edge_levels before set_problem");
		int rc = levels_init(); if (rc) return rc;
		const size_t E = (size_t)S.E;
		long long included = (long long)E;
		if (levels && E > 0) {
			std::vector<unsigned char> h(E);
			for (size_t i = 0; i < E; i++) { h[i] = levels[i] != 0; included -= h[i]; }
			CUDA_TRY(cudaMemcpyAsync(lvLevel.p, h.data(), E, cudaMemcpyHostToDevice, stream));
			g_h2dBytes += (long long)E;
			rc = levels_scatter(); if (rc) return rc;
			if (world > 1 && !comm) included = own_included(h.data());
			CUDA_TRY(cudaStreamSynchronize(stream));      // h dies here
		} else {
			CUDA_TRY(cudaMemsetAsync(lvLevel.p, 0, std::max<size_t>(E, 1), stream));
			rc = levels_scatter(); if (rc) return rc;
			CUDA_TRY(cudaStreamSynchronize(stream));
			if (world > 1 && !comm) included = S.eLocal;
		}
		if (included < 0) return fail(CUBA_ERR_CUDA, "set_edge_levels: reading the shard's edge list failed");
		lvIncluded = included;
		return CUBA_OK;
	}
	// The levels from a device array: normalised and counted on the device; one read-back of the count, which optimize() decides on.
	// Every rank has the whole array: lvIncluded counts all ranks' edges, a CUBA_DRY_SHARD rank its own (as own_included).
	int set_edge_levels_device(const uint8_t* levels, cudaStream_t caller) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "set_edge_levels before set_problem");
		return on_caller_stream(caller, [&] {
			int rc = levels_init(); if (rc) return rc;
			const int E = S.E, eL = S.eLocal, n = std::max(E, eL), nb = (n + RED_BLOCK - 1) / RED_BLOCK;
			CUDA_TRY(lvPartial.alloc(4 * (size_t)std::max(nb, 1))); CUDA_TRY(lvCount.alloc(4));
			if (n > 0) {
				pio::k_levels_in<<<nb, RED_BLOCK, 0, stream>>>(levels, E, e_user.p, eL, lvLevel.p, lvPartial.p);
				launches++;
				CUDA_TRY(cudaGetLastError());
			}
			rc = levels_scatter(); if (rc) return rc;
			lv::k_sum_counts<<<1, RED_BLOCK, 0, stream>>>(lvPartial.p, n > 0 ? nb : 0, lvCount.p);
			launches++;
			CUDA_TRY(cudaGetLastError());
			double included = 0;
			g_d2hBytes += (long long)sizeof(included);
			CUDA_TRY(cudaMemcpyAsync(&included, lvCount.p + (world > 1 && !comm ? 1 : 0), sizeof(included), cudaMemcpyDeviceToHost, stream));
			CUDA_TRY(cudaStreamSynchronize(stream));
			lvIncluded = (long long)included;
			return CUBA_OK;
		});
	}
	// CUBA_DRY_SHARD (no communicator): optimize() and classify_edges see this rank's edges only, so "no edge included" is judged on
	// them alone, on every path.  One read-back of the shard's edge ids, on this diagnostic path only; -1 when it fails.
	long long own_included(const unsigned char* h)
	{
		std::vector<int> u((size_t)S.eLocal);
		if (!u.empty() && cudaMemcpyAsync(u.data(), e_user.p, sizeof(int) * u.size(), cudaMemcpyDeviceToHost, stream) != cudaSuccess) return -1;
		if (cudaStreamSynchronize(stream) != cudaSuccess) return -1;
		long long n = 0;
		for (int v : u) n += h[v] == 0;
		return n;
	}
	int get_edge_levels(uint8_t* out) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "get_edge_levels before set_problem");
		const size_t E = (size_t)S.E;
		if (!lvOn || E == 0) { if (E) memset(out, 0, E); return CUBA_OK; }
		if (world <= 1) {
			CUDA_TRY(cudaMemcpyAsync(out, lvLevel.p, E, cudaMemcpyDeviceToHost, stream));
			CUDA_TRY(cudaStreamSynchronize(stream));
			g_d2hBytes += (long long)E;
			return CUBA_OK;
		}
		int rc = collect_levels(); if (rc) return rc;
		std::vector<double> h(E);
		g_d2hBytes += (long long)(sizeof(double) * E);
		CUDA_TRY(cudaMemcpyAsync(h.data(), chiSq.p, sizeof(double) * E, cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		for (size_t i = 0; i < E; i++) out[i] = h[i] != 0.0;
		return CUBA_OK;
	}
	// landmark-sharded: every rank holds its own edges' levels; the per-edge chi2 path collects them into chiSq (fp64, edge-id order)
	int collect_levels()
	{
		CUDA_TRY(cudaMemsetAsync(chiSq.p, 0, sizeof(double) * (size_t)S.E, stream));
		KLAUNCH(lv::k_levels_out, S.eLocal, e_user.p, lvLevel.p, S.eLocal, chiSq.p);
		return allreduce(chiSq.p, (size_t)S.E, false);
	}
	int get_edge_levels_device(uint8_t* out, cudaStream_t caller) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "get_edge_levels before set_problem");
		const size_t E = (size_t)S.E;
		if (E == 0) return CUBA_OK;
		return on_caller_stream(caller, [&] {
			if (!lvOn) CUDA_TRY(cudaMemsetAsync(out, 0, E, stream));
			else if (world <= 1) CUDA_TRY(cudaMemcpyAsync(out, lvLevel.p, E, cudaMemcpyDeviceToDevice, stream));
			else {
				int rc = collect_levels(); if (rc) return rc;
				KLAUNCH(pio::k_levels_narrow, E, chiSq.p, (int)E, out);
			}
			return CUBA_OK;
		});
	}
	int classify_edges(double chi2Mono, double chi2Stereo, int flags, int32_t* counts) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "classify_edges before set_problem");
		int rc = levels_init(); if (rc) return rc;
		const int eL = S.eLocal, nb = (eL + RED_BLOCK - 1) / RED_BLOCK;
		CUDA_TRY(lvPartial.alloc(4 * (size_t)std::max(nb, 1))); CUDA_TRY(lvCount.alloc(4));
		if (eL > 0) {
			ChiArgs<T> a = chiArgs(cur);
			a.om = e_om0;
			lv::k_classify_edges<T><<<nb, RED_BLOCK, 0, stream>>>(a, e_user.p, lvLevel.p, chi2Mono, chi2Stereo, flags, lvPartial.p);
			launches++;
			CUDA_TRY(cudaGetLastError());
		}
		lv::k_sum_counts<<<1, RED_BLOCK, 0, stream>>>(lvPartial.p, eL > 0 ? nb : 0, lvCount.p);
		launches++;
		CUDA_TRY(cudaGetLastError());
		rc = allreduce(lvCount.p, 4, false); if (rc) return rc;
		double c[4];
		g_d2hBytes += (long long)sizeof(c);
		CUDA_TRY(cudaMemcpyAsync(c, lvCount.p, sizeof(c), cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		// some level changed (on some rank): scatter the mask.  A rank whose own edges kept their levels scatters the same values again.
		if (c[2] + c[3] > 0) {
			rc = levels_scatter(); if (rc) return rc;
		}
		lvIncluded = (long long)(c[0] + c[1]);      // all ranks; under CUBA_DRY_SHARD this rank's own edges, as in set_edge_levels
		if (counts) for (int k = 0; k < 4; k++) counts[k] = (int32_t)c[k];
		return CUBA_OK;
	}

	// ---- structure-only refinement of the held landmarks in place (cuba_landmark_refine.cuh) -----------------------------------
	int num_free_landmarks() const override { return S.numL; }
	bool fp32() const override { return sizeof(T) != 8; }

	// One launch of k_refine_landmarks (after k_check_landmarks for a device list), the counts summed per round and all-reduced, one
	// read-back of the totals and the status word, then the mask scattered once if some level changed.  The list was checked on the
	// host (host list) or is checked on the device (dev).  Host entry: the list goes up, stats / nstats come down, through the batch
	// buffers.
	int optimize_landmarks(const int32_t* list, int n, const pb::Schedule& s, int32_t* counts, cuba_iter_stat* stats, int32_t* nstats,
		bool dev, cudaStream_t caller) override
	{
		if constexpr (sizeof(T) != 8) {
			return fail(CUBA_ERR_INVALID, "optimize_landmarks: the fp32 engine is not supported (use an fp64 or mixed-precision engine)");
		} else {
			if (counts) memset(counts, 0, sizeof(int32_t) * 4 * (size_t)s.n);
			if (n == 0) return CUBA_OK;
			return on_caller_stream(dev ? caller : stream, [&] { return refine_landmarks(list, n, s, counts, stats, nstats, dev); });
		}
	}
	int refine_landmarks(const int32_t* list, int n, const pb::Schedule& s, int32_t* counts, cuba_iter_stat* stats, int32_t* nstats, bool dev)
	{
		int rc = levels_init(); if (rc) return rc;
		const size_t R = (size_t)s.n, nb = (size_t)n, nS = (size_t)s.statOff[s.n];
		const unsigned grid = (unsigned)((nb + ptb::WARPS - 1) / ptb::WARPS);
		CUDA_TRY(lrPartial.alloc(4 * R * grid)); CUDA_TRY(lrTotal.alloc(4 * pb::MAX_ROUNDS + 1));
		int* status = (int*)(lrTotal.p + 4 * R);
		CUDA_TRY(cudaMemsetAsync(lrTotal.p + 4 * R, 0, sizeof(double), stream));
		ptb::LandmarkArgs a;
		a.n = n; a.lmBeg = S.lmBeg; a.lmEnd = S.lmEnd;
		a.pose = pose[cur].p; a.cam = cam.p; a.Xw = Xw[cur].p;
		a.mx = e_mx.p; a.my = e_my.p; a.mz = e_mz.p; a.om0 = e_om0.p; a.ip = e_ip.p; a.user = e_user.p; a.lmPtr = lmPtr.p;
		a.level = lvLevel.p; a.partial = lrPartial.p;
		// per-landmark outputs: the caller's device arrays, or the batch buffers (stats, then nstats) copied down afterwards
		const size_t oN = 4 * nb * nS, nOut = oN + (nb * R + 1) / 2;
		if (dev) {
			a.list = list; a.status = list ? status : nullptr; a.stats = (lm::IterStat*)stats; a.nstats = nstats;
			if (list) {
				CUDA_TRY(lrMark.alloc((size_t)std::max(S.numL, 1)));
				CUDA_TRY(cudaMemsetAsync(lrMark.p, 0, sizeof(int) * (size_t)std::max(S.numL, 1), stream));
				ptb::k_check_landmarks<<<(unsigned)((nb + 255) / 256), 256, 0, stream>>>(list, n, S.numL, lrMark.p, status);
				launches++;
				CUDA_TRY(cudaGetLastError());
			}
		} else {
			a.status = nullptr;
			CUDA_TRY(batchOut.alloc(std::max<size_t>(nOut, 1))); CUDA_TRY(batchHostOut.grow(sizeof(double) * std::max<size_t>(nOut, 1)));
			a.stats = stats ? (lm::IterStat*)batchOut.p : nullptr;
			a.nstats = nstats ? (int*)(batchOut.p + oN) : nullptr;
			a.list = nullptr;
			if (list) {
				const size_t nIn = (nb + 1) / 2;
				CUDA_TRY(batchHostIn.grow(sizeof(double) * nIn)); CUDA_TRY(batchIn.alloc(nIn));
				memcpy(batchHostIn.p, list, sizeof(int32_t) * nb);
				CUDA_TRY(cudaMemcpyAsync(batchIn.p, batchHostIn.p, sizeof(int32_t) * nb, cudaMemcpyHostToDevice, stream));
				g_h2dBytes += (long long)(sizeof(int32_t) * nb);
				a.list = (const int*)batchIn.p;
			}
		}
		ptb::k_refine_landmarks<<<grid, lm::BLOCK, 0, stream>>>(a, s);
		launches++;
		CUDA_TRY(cudaGetLastError());
		for (size_t r = 0; r < R; r++) {
			lv::k_sum_counts<<<1, RED_BLOCK, 0, stream>>>(lrPartial.p + 4 * r * grid, (int)grid, lrTotal.p + 4 * r);
			launches++;
			CUDA_TRY(cudaGetLastError());
		}
		rc = allreduce(lrTotal.p, 4 * R, false); if (rc) return rc;
		double tot[4 * pb::MAX_ROUNDS + 1];
		g_d2hBytes += (long long)(sizeof(double) * (4 * R + 1));
		CUDA_TRY(cudaMemcpyAsync(tot, lrTotal.p, sizeof(double) * (4 * R + 1), cudaMemcpyDeviceToHost, stream));
		const size_t nBack = (stats ? oN : 0) * sizeof(double) + (nstats ? sizeof(int32_t) * nb * R : 0);
		if (!dev && nBack) {
			if (stats) CUDA_TRY(cudaMemcpyAsync(batchHostOut.p, batchOut.p, sizeof(double) * oN, cudaMemcpyDeviceToHost, stream));
			if (nstats) CUDA_TRY(cudaMemcpyAsync((double*)batchHostOut.p + oN, batchOut.p + oN, sizeof(int32_t) * nb * R, cudaMemcpyDeviceToHost, stream));
			g_d2hBytes += (long long)nBack;
		}
		CUDA_TRY(cudaStreamSynchronize(stream));
		int st;
		memcpy(&st, tot + 4 * R, sizeof(st));
		if (st) {
			const bool bad = st & ptb::BAD_INDEX;
			return fail(CUBA_ERR_INVALID, bad ? "optimize_landmarks: a landmark outside [0, numL)" : "optimize_landmarks: a landmark listed twice");
		}
		if (!dev) {
			const double* o = (const double*)batchHostOut.p;
			if (stats) memcpy(stats, o, sizeof(cuba_iter_stat) * nb * nS);
			if (nstats) memcpy(nstats, o + oN, sizeof(int32_t) * nb * R);
		}
		double changed = 0, delta = 0;
		for (size_t r = 0; r < R; r++) {
			changed += tot[4 * r + 2] + tot[4 * r + 3];
			delta += tot[4 * r + 3] - tot[4 * r + 2];
			if (counts) for (int k = 0; k < 4; k++) counts[4 * r + k] = (int32_t)tot[4 * r + k];
		}
		// some level changed (on some rank): scatter the mask once.  The new positions invalidate whatever a trial or a solve left.
		if (changed > 0) { rc = levels_scatter(); if (rc) return rc; }
		lvIncluded += (long long)delta;
		trialValid = false;
		forget_solves();
		return CUBA_OK;
	}

	int get_profile(double* sec) override
	{
		resolveProfile();
		for (int i = 0; i < CUBA_PROF_NUM; i++) sec[i] = prof[i];
		return CUBA_OK;
	}

	// ---- debug getters ---------------------------------------------------------------------------------
	int dbg_hpl_structure(int32_t* colPtr, int32_t* rowInd, int32_t* e2h) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "no problem");
		{ const int rc0 = ensureHostStructure(); if (rc0) return rc0; }
		if (colPtr) memcpy(colPtr, S.hplColPtr.data(), sizeof(int) * S.hplColPtr.size());
		if (rowInd) memcpy(rowInd, S.hplRowInd.data(), sizeof(int) * S.hplRowInd.size());
		if (e2h) memcpy(e2h, S.edge2Hpl.data(), sizeof(int) * S.edge2Hpl.size());
		return CUBA_OK;
	}
	int dbg_hsc_structure(int32_t* rowPtr, int32_t* colInd) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "no problem");
		{ const int rc0 = ensureHostStructure(); if (rc0) return rc0; }
		if (rowPtr) memcpy(rowPtr, S.hscRowPtr.data(), sizeof(int) * S.hscRowPtr.size());
		if (colInd) memcpy(colInd, S.hscColInd.data(), sizeof(int) * S.hscColInd.size());
		return CUBA_OK;
	}
	int download(const T* d, size_t n, double* out)
	{
		std::vector<T> h(n);
		CUDA_TRY(cudaMemcpyAsync(h.data(), d, sizeof(T) * n, cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		for (size_t i = 0; i < n; i++) out[i] = (double)h[i];
		return CUBA_OK;
	}
	int dbg_system(double* oHpp, double* obp, double* oHll, double* obl, double* oHpl) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "no problem");
		int rc;
		if (oHpp && (rc = download(Hpp, 36 * (size_t)S.numP, oHpp))) return rc;
		if (obp && (rc = download(bp, 6 * (size_t)S.numP, obp))) return rc;
		if (oHll && (rc = download(Hll, 9 * (size_t)S.numL, oHll))) return rc;
		if (obl && (rc = download(bl, 3 * (size_t)S.numL, obl))) return rc;
		if (oHpl) {
			// local blocks land at their global positions; foreign blocks read as zero
			memset(oHpl, 0, sizeof(double) * 18 * (size_t)S.nhpl);
			if (stages.mixed) {
				std::vector<float> hf(20 * (size_t)S.nhplLocal);
				CUDA_TRY(cudaMemcpyAsync(hf.data(), HplF.p, sizeof(float) * hf.size(), cudaMemcpyDeviceToHost, stream));
				CUDA_TRY(cudaStreamSynchronize(stream));
				for (size_t b = 0; b < (size_t)S.nhplLocal; b++) for (int e = 0; e < 18; e++) oHpl[18 * ((size_t)S.hplBase + b) + e] = (double)hf[20 * b + e];
			}
			else if ((rc = download(Hpl, 18 * (size_t)S.nhplLocal, oHpl + 18 * (size_t)S.hplBase))) return rc;
		}
		return CUBA_OK;
	}
	int dbg_schur(double* oHsc, double* obsc, double* oinv) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "no problem");
		int rc;
		if ((rc = ensureHostStructure())) return rc;
		if (oHsc) {
			std::vector<double> full(36 * (size_t)S.nfull);
			if ((rc = download(fVal, full.size(), full.data()))) return rc;
			for (int k = 0; k < S.nblk; k++) memcpy(oHsc + 36 * (size_t)k, full.data() + 36 * (size_t)S.u2f[k], sizeof(double) * 36);
		}
		if (obsc && (rc = download(bsc, 6 * (size_t)S.numP, obsc))) return rc;
		if (oinv && (rc = download(invHll, 9 * (size_t)S.numL, oinv))) return rc;
		return CUBA_OK;
	}
	int dbg_delta(double* oxp, double* oxl) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "no problem");
		int rc;
		if (oxp && (rc = download(xp, 6 * (size_t)S.numP, oxp))) return rc;
		if (oxl && (rc = download(xl, 3 * (size_t)S.numL, oxl))) return rc;
		return CUBA_OK;
	}

	int dbg_pcg_timing(long long* out, int maxCtas) override
	{
		const int n = std::min(maxCtas, (int)(pcgTiming.n / 8));     // the last launch sized pcgTiming for its grid
		if (!pcgTiming.p || n <= 0) return 0;
		CUDA_TRY(cudaMemcpyAsync(out, pcgTiming.p, sizeof(long long) * 8 * (size_t)n, cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		return n;
	}

	// include/cuba_b200.h: cuba_debug_get_pcg_info / cuba_debug_get_coarse (host copies; no engine state changes)
	int dbg_pcg_info(int32_t* info, double* coarseLambda) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "no problem");
		CUDA_TRY(cudaStreamSynchronize(stream));
		PcgStatus ps{};
		CUDA_TRY(cudaMemcpy(&ps, &dScal.p->pcg, sizeof(ps), cudaMemcpyDeviceToHost));
		int last = -1, bad = 0;
		if (p5Ok && p5.coarse.A > 0 && p5.coarse.rebuilds > 0) {
			const int nlog = (int)std::min<long long>(p5.coarse.rebuilds, P5_INFO_LOG);
			std::vector<int> log(nlog);
			CUDA_TRY(cudaMemcpy(log.data(), cInfo.p + 1, sizeof(int) * nlog, cudaMemcpyDeviceToHost));
			for (int v : log) if (v != 0) bad++;
			last = log[(int)((p5.coarse.rebuilds - 1) % P5_INFO_LOG)];
		}
		int coarseKernel = CUBA_COARSE_KERNEL_NONE;
		if (lastPcgTwoLevel && lastPcgKernel == CUBA_PCG_KERNEL_PCG4) coarseKernel = coarse_kernel(p4.coarse.A);
		else if (lastPcgTwoLevel && p5Ok) coarseKernel = coarse_kernel(p5.coarse.A);
		const P5Shape& sh = p5.sh;
		const bool tuned = p5Ok && sh.tuned;
		const int32_t v[CUBA_PCG_INFO_LEN] = {
			lastPcgKernel, lastPcgKernel != CUBA_PCG_KERNEL_NONE && lastPcgTwoLevel ? 1 : 0,
			p5Ok ? p5.apc : 0, p5Ok ? p5.G : 0, p5Ok ? p5.gs : 0, p5Ok ? p5.coarse.A : 0,
			p5Ok ? (tuned ? sh.tDims.maxRows : sh.dims.maxRows) : 0, p5Ok ? (tuned ? sh.tDims.capBlocks : sh.dims.capBlocks) : 0,
			p5Ok ? (tuned ? sh.tDims.zhInSmem : sh.dims.zhInSmem) : 0,
			coarseKernel, last, ps.status, ps.iters, (int32_t)p5.coarse.rebuilds, (int32_t)bjRetries, bad };
		if (info) memcpy(info, v, sizeof(v));
		if (coarseLambda) *coarseLambda = p5.coarse.valid ? p5.coarse.lambda : 0.0;
		return CUBA_OK;
	}
	int dbg_coarse(int32_t* rowAgg, double* oAcP, float* oAcInv) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "no problem");
		const CoarseLevel& L = p5.coarse;
		if (!p5Ok || L.A < 1 || !L.valid) return fail(CUBA_ERR_STATE, "debug_get_coarse: no coarse level of k_pcg5 has been built");
		const int A = L.A, nc = 6 * A;
		CUDA_TRY(cudaStreamSynchronize(stream));
		if (rowAgg) {
			std::vector<int> ptr(A + 1);
			CUDA_TRY(cudaMemcpy(ptr.data(), L.aggRow.p, sizeof(int) * (A + 1), cudaMemcpyDeviceToHost));
			for (int i = 0; i < S.numP; i++) rowAgg[i] = -1;
			for (int ag = 0; ag < A; ag++) for (int i = ptr[ag]; i < ptr[ag + 1] && i < S.numP; i++) rowAgg[i] = ag;
		}
		if (oAcP) CUDA_TRY(cudaMemcpy(oAcP, L.AcP.p, sizeof(double) * 36 * ((size_t)A * (A + 1) / 2), cudaMemcpyDeviceToHost));
		if (oAcInv) CUDA_TRY(cudaMemcpy(oAcInv, L.AcInv.p, sizeof(float) * (size_t)nc * nc, cudaMemcpyDeviceToHost));
		return CUBA_OK;
	}
	// include/cuba_b200.h: cuba_debug_coarse_inverse -- k_coarse_dense on a caller's packed matrix, in buffers of its own
	int dbg_coarse_inverse(const double* hAcP, int A, float* hAcInv, int* hInfo) override
	{
		if (A < 1 || !hAcP || !hAcInv || !hInfo) return fail(CUBA_ERR_INVALID, "debug_coarse_inverse: A < 1 or a NULL pointer");
		const size_t nc = 6 * (size_t)A, nblkP = (size_t)A * (A + 1) / 2;
		DBuf<double> dAcP, dT;
		DBuf<float> dInv;
		DBuf<int> dInfo;
		DBuf<GridBar> dBar;
		CUDA_TRY(dAcP.alloc(36 * nblkP)); CUDA_TRY(dInv.alloc(nc * nc)); CUDA_TRY(dInfo.alloc(1)); CUDA_TRY(dBar.alloc(1));
		CUDA_TRY(dT.alloc(cdense::scratch_doubles(A)));
		CUDA_TRY(cudaMemcpyAsync(dAcP.p, hAcP, sizeof(double) * 36 * nblkP, cudaMemcpyHostToDevice, stream));
		CUDA_TRY(cudaMemsetAsync(dBar.p, 0, sizeof(GridBar), stream));
		CUDA_TRY(cudaMemsetAsync(dInfo.p, 0xff, sizeof(int), stream));          // -1 unless the kernel reports
		int rc = launch_coarse_dense(dAcP, A, dT, dInv, dInfo, dBar); if (rc) return rc;
		CUDA_TRY(cudaMemcpyAsync(hAcInv, dInv.p, sizeof(float) * nc * nc, cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaMemcpyAsync(hInfo, dInfo.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		return CUBA_OK;
	}

	// include/cuba_b200.h: cuba_debug_dense_solve -- k_dense_chol (fp64) on a caller's dense matrix, in buffers of its own
	int dbg_dense_solve(const double* hS, const double* hb, int n, double* hx, int* hInfo) override
	{
		if (n < 1 || !hS || !hb || !hx || !hInfo) return fail(CUBA_ERR_INVALID, "debug_dense_solve: n < 1 or a NULL pointer");
		if (n > 6 * dchol::MAX_POSES) return fail(CUBA_ERR_INVALID, "debug_dense_solve: n > " + std::to_string(6 * dchol::MAX_POSES));
		const size_t nn = (size_t)n * n;
		DBuf<double> dS, db, dx, dT, dY;
		DBuf<int> dInfo;
		DBuf<GridBar> dBar;
		CUDA_TRY(dS.upload(hS, nn, stream)); CUDA_TRY(db.upload(hb, (size_t)n, stream)); CUDA_TRY(dx.alloc((size_t)n));
		CUDA_TRY(dT.alloc(dchol::tile_doubles(n))); CUDA_TRY(dY.alloc(dchol::rhs_doubles(n)));
		CUDA_TRY(dInfo.alloc(1)); CUDA_TRY(dBar.alloc(1));
		CUDA_TRY(cudaMemsetAsync(dBar.p, 0, sizeof(GridBar), stream));
		CUDA_TRY(cudaMemsetAsync(dInfo.p, 0xff, sizeof(int), stream));          // -1 unless the kernel reports
		dchol::Args<double> a;
		a.fVal = nullptr; a.blkMap = nullptr; a.dense = dS; a.b = db; a.n = n;
		a.tl = dT; a.y = dY; a.x = dx; a.status = nullptr; a.info = dInfo; a.bar = dBar;
		int rc = launch_dense_chol(a); if (rc) return rc;
		CUDA_TRY(cudaMemcpyAsync(hx, dx.p, sizeof(double) * n, cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaMemcpyAsync(hInfo, dInfo.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
		CUDA_TRY(cudaStreamSynchronize(stream));
		return CUBA_OK;
	}

	// include/cuba_b200.h: cuba_debug_peer_allreduce -- `world` ranks of k_peer_allreduce emulated on this GPU by one cooperative
	// launch of k_peer_allreduce_ranks (numSMs / world CTAs per rank), in buffers of its own
	int dbg_peer_allreduce(int W, size_t n, int calls, const double* parts, double* out) override
	{
		if (W < 1 || W > peer::MAXW || n < 1 || calls < 1 || !parts || !out)
			return fail(CUBA_ERR_INVALID, "debug_peer_allreduce: world outside 1..8, n < 1, calls < 1 or a NULL pointer");
		unsigned int nctas = numSMs / W;
		int perSM = 0;
		CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSM, peer::k_peer_allreduce_ranks<T>, peer::BLOCK, 0));
		if ((long long)perSM * numSMs < (long long)W * nctas)
			return fail(CUBA_ERR_INVALID, "debug_peer_allreduce: " + std::to_string(W * nctas) + " CTAs, but only " + std::to_string(perSM * numSMs) + " can be resident at once");
		// every rank's buffer as launch_peer_allreduce lays it out (n elements, then the signal block), 16-byte aligned
		const size_t sigElems = (2 * peer::MAXW * sizeof(unsigned int) + sizeof(T) - 1) / sizeof(T);
		const size_t stride = (peer_signal_offset(n) + sigElems + 31) / 32 * 32;
		DBuf<T> buf; DBuf<GridBar> bars; DBuf<peer::Args<T>> dArgs;
		CUDA_TRY(buf.alloc(stride * W)); CUDA_TRY(bars.alloc(W));
		CUDA_TRY(cudaMemsetAsync(buf.p, 0, sizeof(T) * stride * W, stream));
		CUDA_TRY(cudaMemsetAsync(bars.p, 0, sizeof(GridBar) * W, stream));
		std::vector<void*> bufs(W);
		for (int r = 0; r < W; r++) bufs[r] = buf.p + stride * r;
		std::vector<peer::Args<T>> ha(W);
		std::vector<T> h((size_t)W * n);
		for (int c = 0; c < calls; c++) {
			// consecutive epochs on the same signal blocks
			for (int r = 0; r < W; r++) ha[r] = peer_args(bufs.data(), r, W, n, (unsigned int)c + 1, bars.p + r);
			CUDA_TRY(dArgs.upload(ha.data(), W, stream));
			for (size_t i = 0; i < (size_t)W * n; i++) h[i] = (T)parts[(size_t)c * W * n + i];
			for (int r = 0; r < W; r++) CUDA_TRY(cudaMemcpyAsync(buf.p + stride * r, h.data() + (size_t)r * n, sizeof(T) * n, cudaMemcpyHostToDevice, stream));
			const peer::Args<T>* pa = dArgs.p;
			void* args[] = { (void*)&pa, (void*)&nctas };
			CUDA_TRY(cudaLaunchCooperativeKernel((void*)peer::k_peer_allreduce_ranks<T>, dim3(W * nctas), dim3(peer::BLOCK), args, 0, stream));
			launches++;
			for (int r = 0; r < W; r++) CUDA_TRY(cudaMemcpyAsync(h.data() + (size_t)r * n, buf.p + stride * r, sizeof(T) * n, cudaMemcpyDeviceToHost, stream));
			CUDA_TRY(cudaStreamSynchronize(stream));
			for (size_t i = 0; i < (size_t)W * n; i++) out[(size_t)c * W * n + i] = (double)h[i];
		}
		return CUBA_OK;
	}

	// include/cuba_b200.h: cuba_debug_pcg5_ranks -- the row-distributed k_pcg5 of a `world`-rank run on the current reduced system,
	// every rank's boards in this GPU's memory and all ranks in one cooperative launch of k_pcg5_ranks, in buffers of its own.  The
	// run is uploaded, laid out, prepared and given its arguments by the engine's own k_pcg5 code (pcg5_upload, Pcg5Run::boards,
	// pcg5_prepare, pcg5_args); only the kernel (k_pcg5_ranks) and where the W board sets live differ from a W-GPU run.
	int dbg_pcg5_ranks(int W, int twoLevel, int nsolves, double* xOut, int32_t* statusOut, int32_t* planOut, int32_t* aggRowOut, float* acInvOut) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "no problem");
		if (W < 1 || W > PCG5_MAXWORLD || nsolves < 1 || !xOut || !statusOut || !planOut)
			return fail(CUBA_ERR_INVALID, "debug_pcg5_ranks: world outside 1..8, nsolves < 1 or a NULL pointer");
		const int numP = S.numP;
		if (numP < 1 || S.numL < 1) return fail(CUBA_ERR_STATE, "debug_pcg5_ranks: no reduced system");
		Pcg5Plan plan;
		build_pcg5_plan(numP, S.nfull, S.fRowPtr, S.fColInd, W, numSMs / W, pcg5_max_agg(), 2 * PCG5_BLOCK / 6, plan, nullptr, 1);
		if (!plan.ok) return fail(CUBA_ERR_INVALID, "debug_pcg5_ranks: no k_pcg5 plan for " + std::to_string(W) + " ranks of " + std::to_string(numSMs / W) + " CTAs");
		P5Shape sh;
		int rc = pcg5_legacy_shape(plan, pcg5_plan_dims(plan, W), W, true, sh); if (rc) return rc;
		const int G = plan.G, nc = 6 * plan.A;
		if ((long long)sh.perSM * numSMs < (long long)W * G)
			return fail(CUBA_ERR_INVALID, "debug_pcg5_ranks: " + std::to_string(W * G) + " CTAs, but only " + std::to_string(sh.perSM * numSMs) + " can be resident at once");
		Pcg5Run R;
		rc = pcg5_upload(R, plan, sh, W, nullptr); if (rc) return rc;
		const size_t nP = (size_t)numP;
		DBuf<T> dZx, dHat, dx;
		DBuf<double> dU, dTiles;
		DBuf<int> dInfo;
		DBuf<GridBar> dBar;
		DBuf<PcgStatus> dStatus;
		DBuf<unsigned long long> boards;
		DBuf<Pcg5Args<T>> dArgs;
		CUDA_TRY(dZx.alloc(36 * nP)); CUDA_TRY(dU.alloc(36 * (size_t)S.nfull)); CUDA_TRY(dHat.alloc(36 * (size_t)S.nfull)); CUDA_TRY(dx.alloc(6 * nP));
		if (twoLevel && coarse_kernel(plan.A) == CUBA_COARSE_KERNEL_DENSE) CUDA_TRY(dTiles.alloc(cdense::scratch_doubles(plan.A)));
		CUDA_TRY(dInfo.alloc(1)); CUDA_TRY(dBar.alloc(1)); CUDA_TRY(dStatus.alloc(W));
		CUDA_TRY(cudaMemsetAsync(R.coarse.AcInv.p, 0, sizeof(float) * (size_t)nc * nc, stream));
		CUDA_TRY(cudaMemsetAsync(dInfo.p, 0, sizeof(int), stream));
		CUDA_TRY(cudaMemsetAsync(dBar.p, 0, sizeof(GridBar), stream));
		// W board sets of the engine's layout, zeroed
		const size_t words = R.boards().words;
		CUDA_TRY(boards.alloc(words * W));
		CUDA_TRY(cudaMemsetAsync(boards.p, 0, sizeof(unsigned long long) * words * W, stream));
		std::vector<unsigned long long*> base(W);
		std::vector<Pcg5Ctl*> ctl(W);
		for (int r = 0; r < W; r++) { base[r] = boards.p + words * r; ctl[r] = R.ctl(base[r]); }
		rc = pcg5_prepare(R, twoLevel != 0, ctl.data(), W, CoarseScratch{ dZx.p, dU.p, dTiles.p, dBar.p }, dInfo.p); if (rc) return rc;
		std::vector<Pcg5Args<T>> ha(W);
		for (int r = 0; r < W; r++) pcg5_args(ha[r], R, twoLevel != 0, r, W, base.data(), dHat.p, dx.p, dStatus.p + r);
		CUDA_TRY(dArgs.upload(ha.data(), W, stream));
		std::vector<T> hx(6 * nP);
		std::vector<PcgStatus> hs(W);
		for (int k = 0; k < nsolves; k++) {
			CUDA_TRY(cudaMemsetAsync(dx.p, 0xff, sizeof(T) * 6 * nP, stream));         // NaN: a row no rank writes stays visible
			const Pcg5Args<T>* pArgs = dArgs.p;
			int g = G;
			void* args[] = { (void*)&pArgs, (void*)&g };
			CUDA_TRY(cudaLaunchCooperativeKernel(sh.fn, dim3(W * G), dim3(PCG5_BLOCK), args, sh.smem, stream));
			for (int r = 0; r < W; r++) k_pcg5_commit<<<1, 1, 0, stream>>>(ctl[r]);
			launches += 1 + W;
			CUDA_TRY(cudaGetLastError());
			CUDA_TRY(cudaMemcpyAsync(hx.data(), dx.p, sizeof(T) * 6 * nP, cudaMemcpyDeviceToHost, stream));
			CUDA_TRY(cudaMemcpyAsync(hs.data(), dStatus.p, sizeof(PcgStatus) * W, cudaMemcpyDeviceToHost, stream));
			CUDA_TRY(cudaStreamSynchronize(stream));
			for (size_t i = 0; i < 6 * nP; i++) xOut[(size_t)k * 6 * nP + i] = (double)hx[i];
			for (int r = 0; r < W; r++) { statusOut[((size_t)k * W + r) * 2] = hs[r].status; statusOut[((size_t)k * W + r) * 2 + 1] = hs[r].iters; }
		}
		int cinfo = 0;
		CUDA_TRY(cudaMemcpy(&cinfo, dInfo.p, sizeof(int), cudaMemcpyDeviceToHost));
		int halo = 0;
		for (unsigned char m : plan.rowPeers) if (m) halo++;
		const int32_t v[8] = { G, plan.gs, plan.A, plan.P.needMax, plan.P.maxRows, halo, sh.big ? 1 : 0, cinfo };
		memcpy(planOut, v, sizeof(v));
		if (aggRowOut) memcpy(aggRowOut, plan.C.aggRow.data(), sizeof(int) * (plan.A + 1));
		if (acInvOut) CUDA_TRY(cudaMemcpy(acInvOut, R.coarse.AcInv.p, sizeof(float) * (size_t)nc * nc, cudaMemcpyDeviceToHost));
		return CUBA_OK;
	}

	// ---- micro-benchmarks --------------------------------------------------------------------------------
	int bench_stage(int stage, int reps, int flush, double lambda, double* ms) override
	{
		if (!haveProblem) return fail(CUBA_ERR_STATE, "bench before set_problem");
		if (reps < 1) reps = 1;
		const size_t flushN = (size_t)40 << 20;   // 320 MB of doubles, several times the 50 MB L2 of an H100
		if (flush) CUDA_TRY(flushBuf.alloc(flushN));
		cudaEvent_t a, b;
		CUDA_TRY(cudaEventCreate(&a)); CUDA_TRY(cudaEventCreate(&b));
		double total = 0;
		const T lam = (T)lambda;
		for (int r = 0; r < reps; r++) {
			if (flush) { k_fill<<<numSMs * 8, 256, 0, stream>>>(flushBuf.p, flushN, (double)r); launches++; }
			CUDA_TRY(cudaEventRecord(a, stream));
			int rc = CUBA_OK;
			switch (stage) {
			case 0: rc = launch_linearize_landmark(); if (!rc) rc = launch_linearize_pose(); break;
			case 1: rc = launch_linearize_landmark(); break;
			case 2: rc = launch_linearize_pose(); break;
			case 3: rc = launch_schur(lam); break;
			case 4: curLambda = lambda; rc = launch_solver(); break;
			case 5: rc = launch_backsub(lam); if (!rc) rc = stage_update_nofetch(lam); break;
			case 6: rc = launch_chi2(cur, 0); break;
			case 7:   // one rebuild of the coarse inverse of k_pcg5 / k_pcg5t (projection, assembly, inverse) from the current system
				if (!p5Ok || p5.coarse.A < 1) rc = fail(CUBA_ERR_STATE, "bench_stage: no two-level k_pcg5 plan");
				else rc = launch_coarse_setup(p5.coarse, coarse_scratch(), p5InfoSlot());
				break;
			default: rc = fail(CUBA_ERR_INVALID, "bench_stage: unknown stage");
			}
			if (rc) return rc;
			CUDA_TRY(cudaEventRecord(b, stream));
			CUDA_TRY(cudaEventSynchronize(b));
			float t = 0;
			CUDA_TRY(cudaEventElapsedTime(&t, a, b));
			total += t;
		}
		cudaEventDestroy(a); cudaEventDestroy(b);
		resolveProfile();
		if (ms) *ms = total / reps;
		return CUBA_OK;
	}
	int stage_update_nofetch(T lam)
	{
		if (S.numP > 0) {
			k_update_poses<T><<<nPoseBlocks, RED_BLOCK, 0, stream>>>(xp, bp, S.numP, lam, pose[cur], pose[cur ^ 1], scalePartialP);
			launches++;
			CUDA_TRY(cudaGetLastError());
		}
		return launch_chi2(cur ^ 1, 1);
	}
};

// ---- the batched LM kernels from host arrays: grow the buffers, pack on the host, copy up, launch, copy down, synchronise, unpack on
// the host
static_assert(sizeof(lm::IterStat) == sizeof(cuba_iter_stat) && sizeof(lm::IterStat) == 32, "cuba_iter_stat layout");

int EngineBase::batch_grow(size_t nIn, size_t nOut)
{
	CUDA_TRY(batchHostIn.grow(sizeof(double) * nIn)); CUDA_TRY(batchHostOut.grow(sizeof(double) * nOut));
	CUDA_TRY(batchIn.alloc(nIn)); CUDA_TRY(batchOut.alloc(nOut));
	return CUBA_OK;
}

// the nIn packed doubles of batchHostIn up to batchIn
int EngineBase::batch_up(size_t nIn)
{
	CUDA_TRY(cudaMemcpyAsync(batchIn.p, batchHostIn.p, sizeof(double) * nIn, cudaMemcpyHostToDevice, stream));
	g_h2dBytes += (long long)(sizeof(double) * nIn);
	return CUBA_OK;
}

// after the one launch on batchIn: the nOut result doubles of batchOut down to batchHostOut, synchronised
int EngineBase::batch_down(size_t nOut)
{
	launches++;
	CUDA_TRY(cudaGetLastError());
	CUDA_TRY(cudaMemcpyAsync(batchHostOut.p, batchOut.p, sizeof(double) * nOut, cudaMemcpyDeviceToHost, stream));
	g_d2hBytes += (long long)(sizeof(double) * nOut);
	CUDA_TRY(cudaStreamSynchronize(stream));
	return CUBA_OK;
}

int EngineBase::optimize_poses(const cuba_pose_batch& bt, const pb::Schedule& s, double* qOut, double* tOut, uint8_t* levelsOut,
	int32_t* counts, cuba_iter_stat* stats, int32_t* nstats)
{
	const size_t B = (size_t)bt.B, nStat = stats ? B * (size_t)s.statOff[s.n] : 0;
	const bio::PoseLayout L(B, (size_t)bt.E2 + (size_t)bt.E3, (size_t)s.n, nStat);
	int rc = batch_grow(L.nIn, L.nOut); if (rc) return rc;
	bio::pack_poses(bt, L, (double*)batchHostIn.p);
	rc = batch_up(L.nIn); if (rc) return rc;
	bio::launch_poses(L, bt.B, s, batchIn.p, batchOut.p, stats != nullptr, stream);
	rc = batch_down(L.nOut); if (rc) return rc;
	const double* o = (const double*)batchHostOut.p;
	const int32_t* p2 = (const int32_t*)((const double*)batchHostIn.p + L.oPtr);
	for (size_t b = 0; b < B; b++) {
		for (int k = 0; k < 4; k++) qOut[4 * b + k] = o[8 * b + k];
		for (int k = 0; k < 3; k++) tOut[3 * b + k] = o[8 * b + 4 + k];
		bio::unpack_rounds(L, o, p2, (int)b, bt.B, s.n, bt.E2, s.statOff[s.n], 0, 1, levelsOut, counts, stats, nstats);
	}
	return CUBA_OK;
}

int EngineBase::optimize_sim3(const cuba_sim3_batch& bt, const s3::Params& p, double* qOut, double* tOut, double* sOut, uint8_t* levelsOut,
	int32_t* ninliers, cuba_iter_stat* stats, int32_t* nstats)
{
	const size_t B = (size_t)bt.B, N = (size_t)bt.N, nStat = stats ? B * (size_t)p.statPer : 0;
	const bio::Sim3Layout L(B, N, nStat);
	int rc = batch_grow(L.nIn, L.nOut); if (rc) return rc;
	bio::pack_sim3(bt, L, (double*)batchHostIn.p);
	rc = batch_up(L.nIn); if (rc) return rc;
	bio::launch_sim3(L, bt.B, p, batchIn.p, batchOut.p, stats != nullptr, stream);
	rc = batch_down(L.nOut); if (rc) return rc;
	const double* o = (const double*)batchHostOut.p;
	for (size_t b = 0; b < B; b++) {
		for (int k = 0; k < 4; k++) qOut[4 * b + k] = o[8 * b + k];
		for (int k = 0; k < 3; k++) tOut[3 * b + k] = o[8 * b + 4 + k];
		sOut[b] = o[8 * b + 7];
	}
	if (stats && nStat) memcpy(stats, o + L.oStat, sizeof(cuba_iter_stat) * nStat);
	const int32_t* oi = (const int32_t*)(o + L.oInt);
	if (ninliers) memcpy(ninliers, oi, sizeof(int32_t) * B);
	if (nstats) memcpy(nstats, oi + B, sizeof(int32_t) * 2 * B);
	if (levelsOut && N) memcpy(levelsOut, (const unsigned char*)(o + L.oLev), N);
	return CUBA_OK;
}

int EngineBase::optimize_points(const cuba_point_batch& bt, const pb::Schedule& s, double* XwOut, uint8_t* levelsOut, int32_t* counts,
	cuba_iter_stat* stats, int32_t* nstats)
{
	const size_t B = (size_t)bt.B, E = (size_t)bt.E2 + (size_t)bt.E3, nStat = stats ? B * (size_t)s.statOff[s.n] : 0;
	const bio::PointLayout L(B, (size_t)bt.P, E, (size_t)s.n, nStat);
	int rc = batch_grow(L.nIn, L.nOut); if (rc) return rc;
	bio::pack_points(bt, L, (double*)batchHostIn.p);
	rc = batch_up(L.nIn); if (rc) return rc;
	bio::launch_points(L, bt.B, E, s, batchIn.p, batchOut.p, stats != nullptr, stream);
	rc = batch_down(L.nOut); if (rc) return rc;
	const double* o = (const double*)batchHostOut.p;
	const int32_t* p2 = (const int32_t*)((const double*)batchHostIn.p + L.oIdx) + E;
	for (size_t b = 0; b < B; b++) {
		for (int k = 0; k < 3; k++) XwOut[3 * b + k] = o[4 * b + k];
		bio::unpack_rounds(L, o, p2, (int)b, bt.B, s.n, bt.E2, s.statOff[s.n], 0, 1, levelsOut, counts, stats, nstats);
	}
	return CUBA_OK;
}

}  // namespace cuba_b200

// ======================================================================================================
// C ABI
// ======================================================================================================
using namespace cuba_b200;

struct cuba_engine { std::unique_ptr<EngineBase> impl; };

extern "C" {

const char* cuba_last_error(void) { return g_err.c_str(); }
int cuba_version(void) { return 100; }

int cuba_engine_create(const cuba_config* cfg, cuba_engine** out)
{
	if (!out) return fail(CUBA_ERR_INVALID, "create: null out");
	cuba_config c;
	memset(&c, 0, sizeof(c));
	c.device = -1; c.deterministic = 1;
	if (cfg) c = *cfg;
	// kernel-selecting slots: a value that names no kernel is an error, not a silent default
	const int r0 = c.reserved[0];
	if (r0 != 0 && (r0 < 2 || r0 > 8))
		return fail(CUBA_ERR_INVALID, "create: reserved[0] = " + std::to_string(r0) + " names no PCG kernel (0, 2..8)");
	StageChoice stages;
	int rc = stage_choice(c, c.use_fp32 != 1, stages); if (rc) return rc;
	std::unique_ptr<EngineBase> impl;
	if (c.use_fp32 == 1) { auto* e = new Engine<float>(); e->cfg = c; impl.reset(e); rc = e->init(); }
	else { auto* e = new Engine<double>(); e->cfg = c; impl.reset(e); rc = e->init(); }
	if (rc) return rc;
	if (getenv("CUBA_NO_STRUCTURE_REUSE")) impl->structureReuse = false;   // like-for-like timing against the reference, which rebuilds everything
	*out = new cuba_engine{ std::move(impl) };
	return CUBA_OK;
}

int cuba_engine_destroy(cuba_engine* e) { delete e; return CUBA_OK; }   // ~Engine switches to its own device itself

#define ENGINE_OR_FAIL(e) if (!(e) || !(e)->impl) return fail(CUBA_ERR_INVALID, "null engine"); DevGuard _devGuard((e)->impl->devOrdinal)

int cuba_engine_set_robust_kernel(cuba_engine* e, int edge_type, int kernel_type, double delta)
{
	ENGINE_OR_FAIL(e);
	if (edge_type < 0 || edge_type > 1 || kernel_type < 0 || kernel_type > 2) return fail(CUBA_ERR_INVALID, "set_robust_kernel: bad type");
	e->impl->rk_type[edge_type] = kernel_type; e->impl->rk_delta[edge_type] = delta;
	return CUBA_OK;
}

int cuba_comm_unique_id(void* out128)
{
	std::string why;
	if (!g_nccl.load(why)) return fail(CUBA_ERR_COMM, why);
	Nccl::UniqueId id;
	const int rc = g_nccl.GetUniqueId(&id);
	if (rc) return fail(CUBA_ERR_COMM, "ncclGetUniqueId failed");
	memcpy(out128, &id, 128);
	return CUBA_OK;
}

int cuba_engine_set_comm(cuba_engine* e, int rank, int world, const void* uid)
{
	ENGINE_OR_FAIL(e);
	if (world < 1 || rank < 0 || rank >= world || world > PCG5_MAXWORLD) return fail(CUBA_ERR_INVALID, "set_comm: bad rank/world (at most 8 ranks)");
	if (e->impl->haveProblem) return fail(CUBA_ERR_STATE, "set_comm must precede set_problem");
	e->impl->rank = rank; e->impl->world = world;
	if (world == 1) return CUBA_OK;
	if (getenv("CUBA_DRY_SHARD")) return CUBA_OK;      // diagnosis: keep the shard, skip every collective (results are then partial sums)
	if (!uid) return fail(CUBA_ERR_INVALID, "set_comm: null unique id");
	std::string why;
	if (!g_nccl.load(why)) return fail(CUBA_ERR_COMM, why);
	Nccl::UniqueId id;
	memcpy(&id, uid, 128);
	const int rc = g_nccl.CommInitRank(&e->impl->comm, world, id, rank);
	if (rc) return fail(CUBA_ERR_COMM, std::string("ncclCommInitRank failed: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?"));
	return CUBA_OK;
}

int cuba_engine_set_problem(cuba_engine* e, const cuba_problem* p) { ENGINE_OR_FAIL(e); return e->impl->set_problem(p); }
int cuba_engine_set_linear_solver(cuba_engine* e, int solver)
{
	// the value first: a bad one is refused before anything (a device included) is touched
	if (solver != CUBA_SOLVER_PCG && solver != CUBA_SOLVER_DENSE_CHOLESKY)
		return fail(CUBA_ERR_INVALID, "set_linear_solver: " + std::to_string(solver) + " names no solver (0 PCG, 1 dense Cholesky)");
	ENGINE_OR_FAIL(e);
	e->impl->linSolver = solver;
	return CUBA_OK;
}
int cuba_engine_set_structure_reuse(cuba_engine* e, int enable) { ENGINE_OR_FAIL(e); e->impl->structureReuse = enable != 0; return CUBA_OK; }
int cuba_engine_get_structure_reuses(cuba_engine* e, long long* count) { ENGINE_OR_FAIL(e); if (count) *count = e->impl->structureReuses; return CUBA_OK; }
int cuba_engine_set_state(cuba_engine* e, const double* q, const double* t, const double* Xw)
{
	ENGINE_OR_FAIL(e);
	if (!q || !t || !Xw) return fail(CUBA_ERR_INVALID, "set_state: null array");
	return e->impl->set_state(q, t, Xw);
}
int cuba_engine_reset_state(cuba_engine* e) { ENGINE_OR_FAIL(e); return e->impl->reset_state(); }
int cuba_engine_get_device(const cuba_engine* e, int* device) { ENGINE_OR_FAIL(e); if (!device) return fail(CUBA_ERR_INVALID, "null out"); *device = e->impl->devOrdinal; return CUBA_OK; }
int cuba_engine_get_stream(cuba_engine* e, void** s) { ENGINE_OR_FAIL(e); if (!s) return fail(CUBA_ERR_INVALID, "null out"); *s = (void*)e->impl->stream; return CUBA_OK; }
int cuba_engine_flush_l2(cuba_engine* e) { ENGINE_OR_FAIL(e); return e->impl->flush_l2(); }
int cuba_engine_get_sizes(const cuba_engine* e, cuba_sizes* out) { ENGINE_OR_FAIL(e); if (!out) return fail(CUBA_ERR_INVALID, "null out"); return e->impl->get_sizes(out); }
int cuba_engine_optimize(cuba_engine* e, int niter, cuba_iter_stat* stats, int* nstats) { ENGINE_OR_FAIL(e); return e->impl->optimize(niter, stats, nstats); }
int cuba_engine_get_state(cuba_engine* e, double* q, double* t, double* Xw) { ENGINE_OR_FAIL(e); return e->impl->get_state(q, t, Xw); }
int cuba_engine_get_chi2(cuba_engine* e, double* per_edge) { ENGINE_OR_FAIL(e); if (!per_edge) return fail(CUBA_ERR_INVALID, "null out"); return e->impl->get_chi2(per_edge); }
int cuba_engine_set_edge_levels(cuba_engine* e, const uint8_t* levels) { ENGINE_OR_FAIL(e); return e->impl->set_edge_levels(levels); }
int cuba_engine_get_edge_levels(cuba_engine* e, uint8_t* levels)
{
	ENGINE_OR_FAIL(e);
	if (!levels) return fail(CUBA_ERR_INVALID, "null out");
	return e->impl->get_edge_levels(levels);
}
int cuba_engine_classify_edges(cuba_engine* e, double chi2_mono, double chi2_stereo, int flags, int32_t* counts)
{
	ENGINE_OR_FAIL(e);
	if (flags & ~(CUBA_CLASSIFY_DEPTH | CUBA_CLASSIFY_REINCLUDE)) return fail(CUBA_ERR_INVALID, "classify_edges: unknown flag");
	return e->impl->classify_edges(chi2_mono, chi2_stereo, flags, counts);
}
// ---- the engine's problem on device-resident arrays: the host entry points' checks and messages, then the work on the engine's
// stream ordered after `stream`'s (NULL: the engine's stream)
int cuba_engine_set_problem_device(cuba_engine* e, const cuba_problem* p_dev, void* stream)
{
	ENGINE_OR_FAIL(e);
	return e->impl->set_problem_device(p_dev, (cudaStream_t)stream);
}
int cuba_engine_set_state_device(cuba_engine* e, const double* q, const double* t, const double* Xw, void* stream)
{
	ENGINE_OR_FAIL(e);
	if (!q || !t || !Xw) return fail(CUBA_ERR_INVALID, "set_state: null array");
	return e->impl->set_state_device(q, t, Xw, (cudaStream_t)stream);
}
int cuba_engine_get_state_device(cuba_engine* e, double* q, double* t, double* Xw, void* stream)
{
	ENGINE_OR_FAIL(e);
	return e->impl->get_state_device(q, t, Xw, (cudaStream_t)stream);
}
int cuba_engine_get_chi2_device(cuba_engine* e, double* per_edge, void* stream)
{
	ENGINE_OR_FAIL(e);
	if (!per_edge) return fail(CUBA_ERR_INVALID, "null out");
	return e->impl->get_chi2_device(per_edge, (cudaStream_t)stream);
}
int cuba_engine_set_edge_levels_device(cuba_engine* e, const uint8_t* levels, void* stream)
{
	ENGINE_OR_FAIL(e);
	return e->impl->set_edge_levels_device(levels, (cudaStream_t)stream);
}
int cuba_engine_get_edge_levels_device(cuba_engine* e, uint8_t* levels, void* stream)
{
	ENGINE_OR_FAIL(e);
	if (!levels) return fail(CUBA_ERR_INVALID, "null out");
	return e->impl->get_edge_levels_device(levels, (cudaStream_t)stream);
}

// The batches of the batched LM kernels come from outside the program: everything a kernel relies on is checked before any work.
// A CSR pointer of B problems over `count` items: present, ptr[0] = 0, non-decreasing and ptr[B] = count (so a negative count
// fails), and every item array present when there are items.
static int csr_ok(const std::string& what, int B, int count, const int32_t* ptr, std::initializer_list<const void*> items)
{
	if (!ptr) return fail(CUBA_ERR_INVALID, what + ": null");
	if (ptr[0] != 0) return fail(CUBA_ERR_INVALID, what + "[0] != 0");
	for (int b = 0; b < B; b++)
		if (ptr[b + 1] < ptr[b]) return fail(CUBA_ERR_INVALID, what + " decreases");
	if (ptr[B] != count) return fail(CUBA_ERR_INVALID, what + "[B] is not the item count");
	for (const void* p : items)
		if (count > 0 && !p) return fail(CUBA_ERR_INVALID, what + ": null item array");
	return CUBA_OK;
}

static bool all_finite(const double* p, size_t n)
{
	for (size_t i = 0; i < n; i++)
		if (!std::isfinite(p[i])) return false;
	return true;
}

// the schedule of optimize_poses / optimize_points (`what`), checked: everything a host can see without the batch
static int pose_schedule(int nrounds, const cuba_pose_round* rounds, pb::Schedule& s, const char* what = "optimize_poses")
{
	if (nrounds < 1 || nrounds > CUBA_POSE_MAX_ROUNDS || !rounds) return fail(CUBA_ERR_INVALID, std::string(what) + ": nrounds outside 1..CUBA_POSE_MAX_ROUNDS");
	static_assert(CUBA_POSE_MAX_ROUNDS == pb::MAX_ROUNDS, "round limit");
	memset(&s, 0, sizeof(s));
	s.n = nrounds;
	long long off = 0;
	for (int r = 0; r < nrounds; r++) {
		const cuba_pose_round& R = rounds[r];
		if (R.iterations < 0) return fail(CUBA_ERR_INVALID, std::string(what) + ": negative iterations");
		if (R.flags & ~(CUBA_CLASSIFY_DEPTH | CUBA_CLASSIFY_REINCLUDE)) return fail(CUBA_ERR_INVALID, std::string(what) + ": unknown flag");
		for (int k = 0; k < 2; k++) {
			if (R.kernel_type[k] < CUBA_ROBUST_NONE || R.kernel_type[k] > CUBA_ROBUST_TUKEY) return fail(CUBA_ERR_INVALID, std::string(what) + ": unknown kernel type");
			if (!std::isfinite(R.delta[k])) return fail(CUBA_ERR_INVALID, std::string(what) + ": non-finite delta");
			s.rk[r].type[k] = R.kernel_type[k]; s.rk[r].delta[k] = R.delta[k];
		}
		s.r[r].iterations = R.iterations; s.r[r].restart = R.restart != 0; s.r[r].flags = R.flags;
		s.r[r].chi2[0] = R.chi2_mono; s.r[r].chi2[1] = R.chi2_stereo;
		s.statOff[r] = (int)off;
		off += R.iterations;
		if (off > INT32_MAX) return fail(CUBA_ERR_INVALID, std::string(what) + ": too many iterations");
	}
	s.statOff[nrounds] = (int)off;
	return CUBA_OK;
}

// the checks of optimize_poses and optimize_poses_device that need no element of the batch's arrays
static int pose_batch_args(const cuba_pose_batch* bt, int nrounds, const cuba_pose_round* rounds, pb::Schedule& s)
{
	if (!bt) return fail(CUBA_ERR_INVALID, "optimize_poses: null batch");
	if (bt->B < 0) return fail(CUBA_ERR_INVALID, "optimize_poses: B < 0");
	return pose_schedule(nrounds, rounds, s);
}

// pose_batch_args' checks of the pointers, for B > 0
static int pose_batch_pointers(const cuba_pose_batch* bt, const double* qOut, const double* tOut)
{
	if (!bt->q || !bt->t || !bt->cam || !qOut || !tOut) return fail(CUBA_ERR_INVALID, "optimize_poses: null pose array");
	if ((long long)bt->E2 + bt->E3 > INT32_MAX) return fail(CUBA_ERR_INVALID, "optimize_poses: too many edges");
	return CUBA_OK;
}

int cuba_engine_optimize_poses(cuba_engine* e, const cuba_pose_batch* bt, int nrounds, const cuba_pose_round* rounds,
	double* q_out, double* t_out, uint8_t* levels_out, int32_t* counts, cuba_iter_stat* stats, int32_t* nstats)
{
	ENGINE_OR_FAIL(e);
	pb::Schedule s;
	int rc = pose_batch_args(bt, nrounds, rounds, s); if (rc) return rc;
	const int B = bt->B;
	if (B == 0) return CUBA_OK;
	rc = pose_batch_pointers(bt, q_out, t_out); if (rc) return rc;
	rc = csr_ok("optimize_poses: ptr2", B, bt->E2, bt->ptr2, { bt->X2, bt->meas2, bt->omega2 }); if (rc) return rc;
	rc = csr_ok("optimize_poses: ptr3", B, bt->E3, bt->ptr3, { bt->X3, bt->meas3, bt->omega3 }); if (rc) return rc;
	if (!all_finite(bt->omega2, bt->E2) || !all_finite(bt->omega3, bt->E3)) return fail(CUBA_ERR_INVALID, "optimize_poses: non-finite omega");
	return e->impl->optimize_poses(*bt, s, q_out, t_out, levels_out, counts, stats, nstats);
}

// host arrays of a point batch: a pose index outside [0, P)
static bool poses_in_range(const int32_t* iP, int n, int P)
{
	for (int i = 0; i < n; i++)
		if (iP[i] < 0 || iP[i] >= P) return false;
	return true;
}

// the checks of optimize_points and optimize_points_device that need no element of the batch's arrays
static int point_batch_args(const cuba_point_batch* bt, int nrounds, const cuba_pose_round* rounds, pb::Schedule& s)
{
	if (!bt) return fail(CUBA_ERR_INVALID, "optimize_points: null batch");
	if (bt->B < 0) return fail(CUBA_ERR_INVALID, "optimize_points: B < 0");
	if (bt->P < 0) return fail(CUBA_ERR_INVALID, "optimize_points: P < 0");
	if (bt->E2 < 0) return fail(CUBA_ERR_INVALID, "optimize_points: E2 < 0");
	if (bt->E3 < 0) return fail(CUBA_ERR_INVALID, "optimize_points: E3 < 0");
	return pose_schedule(nrounds, rounds, s, "optimize_points");
}

// point_batch_args' checks of the pointers, for B > 0
static int point_batch_pointers(const cuba_point_batch* bt, const double* XwOut)
{
	if (!bt->Xw || !XwOut) return fail(CUBA_ERR_INVALID, "optimize_points: null Xw");
	if (bt->P > 0 && (!bt->q || !bt->t || !bt->cam)) return fail(CUBA_ERR_INVALID, "optimize_points: null pose array");
	if ((long long)bt->E2 + bt->E3 > INT32_MAX) return fail(CUBA_ERR_INVALID, "optimize_points: too many edges");
	return CUBA_OK;
}

int cuba_engine_optimize_points(cuba_engine* e, const cuba_point_batch* bt, int nrounds, const cuba_pose_round* rounds, double* Xw_out,
	uint8_t* levels_out, int32_t* counts, cuba_iter_stat* stats, int32_t* nstats)
{
	ENGINE_OR_FAIL(e);
	pb::Schedule s;
	int rc = point_batch_args(bt, nrounds, rounds, s); if (rc) return rc;
	const int B = bt->B;
	if (B == 0) return CUBA_OK;
	rc = point_batch_pointers(bt, Xw_out); if (rc) return rc;
	rc = csr_ok("optimize_points: ptr2", B, bt->E2, bt->ptr2, { bt->iP2, bt->meas2, bt->omega2 }); if (rc) return rc;
	rc = csr_ok("optimize_points: ptr3", B, bt->E3, bt->ptr3, { bt->iP3, bt->meas3, bt->omega3 }); if (rc) return rc;
	if (!poses_in_range(bt->iP2, bt->E2, bt->P)) return fail(CUBA_ERR_INVALID, "optimize_points: iP2 outside [0, P)");
	if (!poses_in_range(bt->iP3, bt->E3, bt->P)) return fail(CUBA_ERR_INVALID, "optimize_points: iP3 outside [0, P)");
	if (!all_finite(bt->omega2, bt->E2) || !all_finite(bt->omega3, bt->E3)) return fail(CUBA_ERR_INVALID, "optimize_points: non-finite omega");
	return e->impl->optimize_points(*bt, s, Xw_out, levels_out, counts, stats, nstats);
}

// the parameters of optimize_sim3, checked
static int sim3_params(const cuba_sim3_params& P, s3::Params& p)
{
	if (!std::isfinite(P.chi2) || !(P.chi2 > 0)) return fail(CUBA_ERR_INVALID, "optimize_sim3: chi2 not finite and positive");
	if (P.iterations < 0 || P.iterations_bad < 0 || P.iterations_good < 0) return fail(CUBA_ERR_INVALID, "optimize_sim3: negative iterations");
	if (P.min_pairs < 0) return fail(CUBA_ERR_INVALID, "optimize_sim3: negative min_pairs");
	if ((long long)P.iterations + std::max(P.iterations_bad, P.iterations_good) > INT32_MAX)
		return fail(CUBA_ERR_INVALID, "optimize_sim3: too many iterations");
	p.chi2 = P.chi2; p.delta = std::sqrt(P.chi2);
	p.iterations = P.iterations; p.iterationsBad = P.iterations_bad; p.iterationsGood = P.iterations_good; p.minPairs = P.min_pairs;
	p.statPer = P.iterations + std::max(P.iterations_bad, P.iterations_good);
	return CUBA_OK;
}

// the checks of optimize_sim3 and optimize_sim3_device that need no element of the batch's arrays
static int sim3_batch_args(const cuba_sim3_batch* bt, const cuba_sim3_params* params, s3::Params& p)
{
	if (!bt || !params) return fail(CUBA_ERR_INVALID, "optimize_sim3: null batch or params");
	const int rc = sim3_params(*params, p); if (rc) return rc;
	if (bt->B < 0) return fail(CUBA_ERR_INVALID, "optimize_sim3: B < 0");
	if (bt->N < 0) return fail(CUBA_ERR_INVALID, "optimize_sim3: N < 0");
	return CUBA_OK;
}

// sim3_batch_args' checks of the problem pointers, for B > 0
static int sim3_batch_pointers(const cuba_sim3_batch* bt, const double* qOut, const double* tOut, const double* sOut)
{
	if (!bt->q || !bt->t || !bt->s || !bt->cam1 || !bt->cam2 || !qOut || !tOut || !sOut)
		return fail(CUBA_ERR_INVALID, "optimize_sim3: null problem array");
	return CUBA_OK;
}

int cuba_engine_optimize_sim3(cuba_engine* e, const cuba_sim3_batch* bt, const cuba_sim3_params* params, double* q_out, double* t_out,
	double* s_out, uint8_t* levels_out, int32_t* ninliers, cuba_iter_stat* stats, int32_t* nstats)
{
	ENGINE_OR_FAIL(e);
	s3::Params p;
	int rc = sim3_batch_args(bt, params, p); if (rc) return rc;
	const int B = bt->B;
	if (B == 0) return CUBA_OK;
	const size_t nb = (size_t)B, N = (size_t)bt->N;
	rc = csr_ok("optimize_sim3: ptr", B, bt->N, bt->ptr, { bt->X1, bt->X2, bt->obs1, bt->obs2, bt->omega1, bt->omega2 }); if (rc) return rc;
	rc = sim3_batch_pointers(bt, q_out, t_out, s_out); if (rc) return rc;
	if (!all_finite(bt->q, 4 * nb) || !all_finite(bt->t, 3 * nb) || !all_finite(bt->s, nb) || !all_finite(bt->cam1, 4 * nb) ||
		!all_finite(bt->cam2, 4 * nb))
		return fail(CUBA_ERR_INVALID, "optimize_sim3: non-finite S12 or intrinsics");
	for (size_t b = 0; b < nb; b++)
		if (!(bt->s[b] > 0)) return fail(CUBA_ERR_INVALID, "optimize_sim3: s <= 0");
	if (!all_finite(bt->X1, 3 * N) || !all_finite(bt->X2, 3 * N) || !all_finite(bt->obs1, 2 * N) || !all_finite(bt->obs2, 2 * N) ||
		!all_finite(bt->omega1, N) || !all_finite(bt->omega2, N))
		return fail(CUBA_ERR_INVALID, "optimize_sim3: non-finite pair");
	return e->impl->optimize_sim3(*bt, p, q_out, t_out, s_out, levels_out, ninliers, stats, nstats);
}

// ---- the batches on device-resident data (cuba_batch_io.cuh).  Host-side checks come first and touch neither the engine nor a
// device; the data checks run on the device into *status.

// csr_ok's checks that need no element of ptr
static int csr_present(const std::string& what, int count, const int32_t* ptr, std::initializer_list<const void*> items)
{
	if (!ptr) return fail(CUBA_ERR_INVALID, what + ": null");
	if (count < 0) return fail(CUBA_ERR_INVALID, what + "[B] is not the item count");
	for (const void* p : items)
		if (count > 0 && !p) return fail(CUBA_ERR_INVALID, what + ": null item array");
	return CUBA_OK;
}

static int workspace_ok(const char* what, const void* ws, size_t bytes, size_t need)
{
	if (bytes < need || (need > 0 && !ws))
		return fail(CUBA_ERR_INVALID, std::string(what) + ": workspace of " + std::to_string(bytes) + " bytes, " + std::to_string(need) + " needed");
	if ((uintptr_t)ws % alignof(double)) return fail(CUBA_ERR_INVALID, std::string(what) + ": workspace not 8-byte aligned");
	return CUBA_OK;
}

// keeps the last error as it was over its scope: a size query leaves it alone
struct KeepLastError {
	const std::string saved = g_err;
	~KeepLastError() { g_err = saved; }
};

static cudaStream_t batch_stream(cuba_engine* e, void* stream) { return stream ? (cudaStream_t)stream : e->impl->stream; }

static size_t pose_workspace(int B, int E2, int E3, const pb::Schedule& s, bool withStats)
{
	const size_t nb = (size_t)B;
	const bio::PoseLayout L(nb, (size_t)E2 + (size_t)E3, (size_t)s.n, withStats ? nb * (size_t)s.statOff[s.n] : 0);
	return sizeof(double) * (L.nIn + L.nOut);
}

size_t cuba_pose_batch_workspace_bytes(int B, int E2, int E3, int nrounds, const cuba_pose_round* rounds, int with_stats)
{
	pb::Schedule s;
	if (B <= 0 || E2 < 0 || E3 < 0 || (long long)E2 + E3 > INT32_MAX) return 0;
	KeepLastError keep;
	return pose_schedule(nrounds, rounds, s) ? 0 : pose_workspace(B, E2, E3, s, with_stats != 0);
}

int cuba_engine_optimize_poses_device(cuba_engine* e, const cuba_pose_batch* bt, int nrounds, const cuba_pose_round* rounds,
	void* workspace, size_t workspace_bytes, double* q_out, double* t_out, uint8_t* levels_out, int32_t* counts, cuba_iter_stat* stats,
	int32_t* nstats, int32_t* status, void* stream)
{
	pb::Schedule s;
	int rc = pose_batch_args(bt, nrounds, rounds, s); if (rc) return rc;
	if (!status) return fail(CUBA_ERR_INVALID, "optimize_poses_device: null status");
	const int B = bt->B;
	if (B > 0) {
		rc = pose_batch_pointers(bt, q_out, t_out); if (rc) return rc;
		rc = csr_present("optimize_poses: ptr2", bt->E2, bt->ptr2, { bt->X2, bt->meas2, bt->omega2 }); if (rc) return rc;
		rc = csr_present("optimize_poses: ptr3", bt->E3, bt->ptr3, { bt->X3, bt->meas3, bt->omega3 }); if (rc) return rc;
		rc = workspace_ok("optimize_poses_device", workspace, workspace_bytes, pose_workspace(B, bt->E2, bt->E3, s, stats != nullptr)); if (rc) return rc;
	}
	ENGINE_OR_FAIL(e);
	const cudaStream_t st = batch_stream(e, stream);
	CUDA_TRY(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
	if (B == 0) return CUBA_OK;
	const size_t nb = (size_t)B, E = (size_t)bt->E2 + (size_t)bt->E3, statPer = (size_t)s.statOff[s.n];
	const bio::PoseLayout L(nb, E, (size_t)s.n, stats ? nb * statPer : 0);
	double* in = (double*)workspace;
	bio::k_validate_poses<<<bio::grid_for(std::max(nb + 1, E)), bio::BLOCK, 0, st>>>(*bt, status);
	bio::k_pack_poses<<<(unsigned)B, bio::BLOCK, 0, st>>>(*bt, L, in, status);
	bio::launch_poses(L, B, s, in, in + L.nIn, stats != nullptr, st);
	bio::k_unpack_poses<<<(unsigned)B, bio::BLOCK, 0, st>>>(L, B, s.n, bt->E2, (int)statPer, in, q_out, t_out, levels_out, counts, stats, nstats, status);
	CUDA_TRY(cudaGetLastError());
	return CUBA_OK;
}

static size_t sim3_workspace(int B, int N, const s3::Params& p, bool withStats)
{
	const bio::Sim3Layout L((size_t)B, (size_t)N, withStats ? (size_t)B * (size_t)p.statPer : 0);
	return sizeof(double) * (L.nIn + L.nOut);
}

size_t cuba_sim3_batch_workspace_bytes(int B, int N, const cuba_sim3_params* params, int with_stats)
{
	s3::Params p;
	if (B <= 0 || N < 0 || !params) return 0;
	KeepLastError keep;
	return sim3_params(*params, p) ? 0 : sim3_workspace(B, N, p, with_stats != 0);
}

int cuba_engine_optimize_sim3_device(cuba_engine* e, const cuba_sim3_batch* bt, const cuba_sim3_params* params,
	void* workspace, size_t workspace_bytes, double* q_out, double* t_out, double* s_out, uint8_t* levels_out, int32_t* ninliers,
	cuba_iter_stat* stats, int32_t* nstats, int32_t* status, void* stream)
{
	s3::Params p;
	int rc = sim3_batch_args(bt, params, p); if (rc) return rc;
	if (!status) return fail(CUBA_ERR_INVALID, "optimize_sim3_device: null status");
	const int B = bt->B;
	if (B > 0) {
		rc = csr_present("optimize_sim3: ptr", bt->N, bt->ptr, { bt->X1, bt->X2, bt->obs1, bt->obs2, bt->omega1, bt->omega2 }); if (rc) return rc;
		rc = sim3_batch_pointers(bt, q_out, t_out, s_out); if (rc) return rc;
		rc = workspace_ok("optimize_sim3_device", workspace, workspace_bytes, sim3_workspace(B, bt->N, p, stats != nullptr)); if (rc) return rc;
	}
	ENGINE_OR_FAIL(e);
	const cudaStream_t st = batch_stream(e, stream);
	CUDA_TRY(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
	if (B == 0) return CUBA_OK;
	const size_t nb = (size_t)B, N = (size_t)bt->N, nStat = stats ? nb * (size_t)p.statPer : 0;
	const bio::Sim3Layout L(nb, N, nStat);
	double* in = (double*)workspace;
	bio::k_validate_sim3<<<bio::grid_for(std::max(4 * nb + 1, 3 * N)), bio::BLOCK, 0, st>>>(*bt, status);
	bio::k_pack_sim3<<<bio::grid_for(s3::PROB * nb + s3::PAIR * N + nb + 1), bio::BLOCK, 0, st>>>(*bt, L, in, status);
	bio::launch_sim3(L, B, p, in, in + L.nIn, stats != nullptr, st);
	bio::k_unpack_sim3<<<bio::grid_for(std::max(8 * nb, std::max(4 * nStat, N))), bio::BLOCK, 0, st>>>(L, B, bt->N, nStat, in, q_out, t_out,
		s_out, levels_out, ninliers, stats, nstats, status);
	CUDA_TRY(cudaGetLastError());
	return CUBA_OK;
}

static size_t point_workspace(int B, int P, int E2, int E3, const pb::Schedule& s, bool withStats)
{
	const size_t nb = (size_t)B;
	const bio::PointLayout L(nb, (size_t)P, (size_t)E2 + (size_t)E3, (size_t)s.n, withStats ? nb * (size_t)s.statOff[s.n] : 0);
	return sizeof(double) * (L.nIn + L.nOut);
}

size_t cuba_point_batch_workspace_bytes(int B, int P, int E2, int E3, int nrounds, const cuba_pose_round* rounds, int with_stats)
{
	pb::Schedule s;
	if (B <= 0 || P < 0 || E2 < 0 || E3 < 0 || (long long)E2 + E3 > INT32_MAX) return 0;
	KeepLastError keep;
	return pose_schedule(nrounds, rounds, s) ? 0 : point_workspace(B, P, E2, E3, s, with_stats != 0);
}

int cuba_engine_optimize_points_device(cuba_engine* e, const cuba_point_batch* bt, int nrounds, const cuba_pose_round* rounds,
	void* workspace, size_t workspace_bytes, double* Xw_out, uint8_t* levels_out, int32_t* counts, cuba_iter_stat* stats,
	int32_t* nstats, int32_t* status, void* stream)
{
	pb::Schedule s;
	int rc = point_batch_args(bt, nrounds, rounds, s); if (rc) return rc;
	if (!status) return fail(CUBA_ERR_INVALID, "optimize_points_device: null status");
	const int B = bt->B;
	if (B > 0) {
		rc = point_batch_pointers(bt, Xw_out); if (rc) return rc;
		rc = csr_present("optimize_points: ptr2", bt->E2, bt->ptr2, { bt->iP2, bt->meas2, bt->omega2 }); if (rc) return rc;
		rc = csr_present("optimize_points: ptr3", bt->E3, bt->ptr3, { bt->iP3, bt->meas3, bt->omega3 }); if (rc) return rc;
		rc = workspace_ok("optimize_points_device", workspace, workspace_bytes, point_workspace(B, bt->P, bt->E2, bt->E3, s, stats != nullptr)); if (rc) return rc;
	}
	ENGINE_OR_FAIL(e);
	const cudaStream_t st = batch_stream(e, stream);
	CUDA_TRY(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
	if (B == 0) return CUBA_OK;
	const size_t nb = (size_t)B, E = (size_t)bt->E2 + (size_t)bt->E3, statPer = (size_t)s.statOff[s.n];
	const bio::PointLayout L(nb, (size_t)bt->P, E, (size_t)s.n, stats ? nb * statPer : 0);
	double* in = (double*)workspace;
	const unsigned gridIo = (unsigned)((nb + bio::POINTS_PER_BLOCK - 1) / bio::POINTS_PER_BLOCK);
	bio::k_validate_points<<<bio::grid_for(std::max(nb + 1, E)), bio::BLOCK, 0, st>>>(*bt, status);
	bio::k_pack_points<<<gridIo, bio::BLOCK, 0, st>>>(*bt, L, in, status);
	bio::launch_points(L, B, E, s, in, in + L.nIn, stats != nullptr, st);
	bio::k_unpack_points<<<gridIo, bio::BLOCK, 0, st>>>(L, B, s.n, bt->E2, bt->E3, (int)statPer, in, Xw_out, levels_out, counts, stats, nstats, status);
	CUDA_TRY(cudaGetLastError());
	return CUBA_OK;
}

// The checks of optimize_landmarks and optimize_landmarks_device that need no list entry, in the order the header states them
static int landmark_args(cuba_engine* e, const int32_t* landmarks, int32_t n, int nrounds, const cuba_pose_round* rounds, pb::Schedule& s)
{
	int rc = pose_schedule(nrounds, rounds, s, "optimize_points"); if (rc) return rc;
	if (n < 0) return fail(CUBA_ERR_INVALID, "optimize_landmarks: n < 0");
	if (!e->impl->haveProblem) return fail(CUBA_ERR_STATE, "optimize_landmarks before set_problem");
	if (!landmarks && n != e->impl->num_free_landmarks()) return fail(CUBA_ERR_INVALID, "optimize_landmarks: a NULL list needs n = numL");
	return CUBA_OK;
}

int cuba_engine_optimize_landmarks(cuba_engine* e, const int32_t* landmarks, int32_t n, int nrounds, const cuba_pose_round* rounds,
	int32_t* counts, cuba_iter_stat* stats, int32_t* nstats)
{
	ENGINE_OR_FAIL(e);
	pb::Schedule s;
	int rc = landmark_args(e, landmarks, n, nrounds, rounds, s); if (rc) return rc;
	if (landmarks) {
		const int numL = e->impl->num_free_landmarks();
		std::vector<unsigned char> seen((size_t)std::max(numL, 1), 0);
		for (int32_t i = 0; i < n; i++) {
			const int32_t l = landmarks[i];
			if (l < 0 || l >= numL) return fail(CUBA_ERR_INVALID, "optimize_landmarks: landmarks[" + std::to_string(i) + "] outside [0, numL)");
			if (seen[(size_t)l]++) return fail(CUBA_ERR_INVALID, "optimize_landmarks: landmarks[" + std::to_string(i) + "] listed twice");
		}
	}
	if (e->impl->fp32()) return fail(CUBA_ERR_INVALID, "optimize_landmarks: the fp32 engine is not supported (use an fp64 or mixed-precision engine)");
	return e->impl->optimize_landmarks(landmarks, n, s, counts, stats, nstats, false, nullptr);
}

int cuba_engine_optimize_landmarks_device(cuba_engine* e, const int32_t* landmarks, int32_t n, int nrounds, const cuba_pose_round* rounds,
	int32_t* counts, cuba_iter_stat* stats, int32_t* nstats, void* stream)
{
	ENGINE_OR_FAIL(e);
	pb::Schedule s;
	int rc = landmark_args(e, landmarks, n, nrounds, rounds, s); if (rc) return rc;
	if (e->impl->fp32()) return fail(CUBA_ERR_INVALID, "optimize_landmarks: the fp32 engine is not supported (use an fp64 or mixed-precision engine)");
	return e->impl->optimize_landmarks(landmarks, n, s, counts, stats, nstats, true, (cudaStream_t)stream);
}

int cuba_engine_get_profile(cuba_engine* e, double* sec) { ENGINE_OR_FAIL(e); if (!sec) return fail(CUBA_ERR_INVALID, "null out"); return e->impl->get_profile(sec); }
// debug: per-CTA phase timings of the last PCG launch (library built with -DCUBA_PCG_TIMING); returns the CTA count
int cuba_debug_get_pcg_timing(cuba_engine* e, long long* out, int maxCtas)
{
	if (!e || !e->impl) return -1;
	DevGuard guard(e->impl->devOrdinal);
	return e->impl->dbg_pcg_timing(out, maxCtas);
}
int cuba_get_transfer_bytes(long long* h2d, long long* d2h) { if (h2d) *h2d = g_h2dBytes; if (d2h) *d2h = g_d2hBytes; return CUBA_OK; }
int cuba_engine_get_launch_count(cuba_engine* e, long long* count) { ENGINE_OR_FAIL(e); if (count) *count = e->impl->launches; return CUBA_OK; }

int cuba_stage_linearize(cuba_engine* e, double* chi2) { ENGINE_OR_FAIL(e); return e->impl->stage_linearize(chi2); }
int cuba_stage_max_diagonal(cuba_engine* e, double* md) { ENGINE_OR_FAIL(e); return e->impl->stage_max_diagonal(md); }
int cuba_stage_solve(cuba_engine* e, double lambda, int* iters, int* ok)
{
	ENGINE_OR_FAIL(e);
	int it = 0, k = 1;
	const int rc = e->impl->stage_solve(lambda, &it, &k);
	if (iters) *iters = it;
	if (ok) *ok = k;
	return rc;
}
int cuba_stage_update(cuba_engine* e, double lambda, double* chi, double* scale) { ENGINE_OR_FAIL(e); return e->impl->stage_update(lambda, chi, scale); }
int cuba_stage_commit(cuba_engine* e, int accept) { ENGINE_OR_FAIL(e); return e->impl->stage_commit(accept); }
int cuba_stage_chi2(cuba_engine* e, double* chi) { ENGINE_OR_FAIL(e); return e->impl->stage_chi2(chi); }

int cuba_debug_get_hpl_structure(cuba_engine* e, int32_t* colPtr, int32_t* rowInd, int32_t* e2h) { ENGINE_OR_FAIL(e); return e->impl->dbg_hpl_structure(colPtr, rowInd, e2h); }
int cuba_debug_get_hsc_structure(cuba_engine* e, int32_t* rowPtr, int32_t* colInd) { ENGINE_OR_FAIL(e); return e->impl->dbg_hsc_structure(rowPtr, colInd); }
int cuba_debug_get_system(cuba_engine* e, double* Hpp, double* bp, double* Hll, double* bl, double* Hpl) { ENGINE_OR_FAIL(e); return e->impl->dbg_system(Hpp, bp, Hll, bl, Hpl); }
int cuba_debug_get_schur(cuba_engine* e, double* Hsc, double* bsc, double* invHll) { ENGINE_OR_FAIL(e); return e->impl->dbg_schur(Hsc, bsc, invHll); }
int cuba_debug_get_delta(cuba_engine* e, double* xp, double* xl) { ENGINE_OR_FAIL(e); return e->impl->dbg_delta(xp, xl); }
int cuba_debug_get_pcg_info(cuba_engine* e, int32_t* info, double* coarse_lambda) { ENGINE_OR_FAIL(e); return e->impl->dbg_pcg_info(info, coarse_lambda); }
int cuba_debug_get_coarse(cuba_engine* e, int32_t* aggRow, double* AcP, float* AcInv) { ENGINE_OR_FAIL(e); return e->impl->dbg_coarse(aggRow, AcP, AcInv); }
int cuba_debug_coarse_inverse(cuba_engine* e, const double* AcP, int A, float* AcInv, int* info) { ENGINE_OR_FAIL(e); return e->impl->dbg_coarse_inverse(AcP, A, AcInv, info); }
int cuba_debug_dense_solve(cuba_engine* e, const double* S, const double* b, int n, double* x, int* info) { ENGINE_OR_FAIL(e); return e->impl->dbg_dense_solve(S, b, n, x, info); }
int cuba_debug_peer_allreduce(cuba_engine* e, int world, int64_t n, int calls, const double* parts, double* out)
{
	ENGINE_OR_FAIL(e);
	if (n < 1) return fail(CUBA_ERR_INVALID, "debug_peer_allreduce: n < 1");
	return e->impl->dbg_peer_allreduce(world, (size_t)n, calls, parts, out);
}
int cuba_debug_pcg5_ranks(cuba_engine* e, int world, int two_level, int nsolves, double* x, int32_t* status, int32_t* plan, int32_t* aggRow, float* AcInv)
{
	ENGINE_OR_FAIL(e);
	return e->impl->dbg_pcg5_ranks(world, two_level, nsolves, x, status, plan, aggRow, AcInv);
}
int cuba_debug_build_structure_host(const cuba_problem* p, int rank, int world, cuba_sizes* sizes,
	int32_t* hplColPtr, int32_t* hplRowInd, int32_t* edge2Hpl, int32_t* hscRowPtr, int32_t* hscColInd,
	int32_t* fullRowPtr, int32_t* fullColInd, int32_t* shard)
{
	if (!p) return fail(CUBA_ERR_INVALID, "null problem");
	Structure S;
	const char* err = "";
	if (!build_structure(p->Pall, p->numP, p->Lall, p->numL, p->E2, p->idx2, p->E3, p->idx3, rank, world, TILE, S, &err))
		return fail(CUBA_ERR_INVALID, err);
	if (sizes) {
		sizes->Pall = S.Pall; sizes->numP = S.numP; sizes->Lall = S.Lall; sizes->numL = S.numL; sizes->E2 = S.E2; sizes->E3 = S.E3;
		sizes->nhpl = S.nhpl; sizes->nblk = S.nblk; sizes->nmul = (int32_t)S.nmul; sizes->nblk_full = S.nfull;
	}
	auto cp = [](int32_t* dst, const std::vector<int>& v) { if (dst && !v.empty()) memcpy(dst, v.data(), sizeof(int) * v.size()); };
	cp(hplColPtr, S.hplColPtr); cp(hplRowInd, S.hplRowInd); cp(edge2Hpl, S.edge2Hpl);
	cp(hscRowPtr, S.hscRowPtr); cp(hscColInd, S.hscColInd); cp(fullRowPtr, S.fRowPtr); cp(fullColInd, S.fColInd);
	if (shard) { shard[0] = S.lmBeg; shard[1] = S.lmEnd; shard[2] = S.eLocal; shard[3] = (int32_t)S.nmulLocal; }
	// internal consistency (cheap): tiles cover the shard, products reference blocks of one landmark with row(i)<=row(j), and
	// with i<=j except between two blocks of one pose
	if ((int)S.tileLm.size() < 1 || S.tileLm.front() != S.lmBeg || S.tileLm.back() != S.lmEnd) return fail(CUBA_ERR_INVALID, "structure self-check: tiles");
	for (size_t t = 0; t + 1 < S.tileLm.size(); t++) {
		const int nl = S.tileLm[t + 1] - S.tileLm[t];
		const int ne = S.lmPtr[S.tileLm[t + 1]] - S.lmPtr[S.tileLm[t]];
		if (nl < 1 || nl > TILE || (ne > TILE && nl != 1)) return fail(CUBA_ERR_INVALID, "structure self-check: tile size");
	}
	for (int k = 0; k < S.nblk; k++)
		for (int n = S.prodPtr[k]; n < S.prodPtr[k + 1]; n++) {
			const int i = S.prodI[n] + S.hplBase, j = S.prodJ[n] + S.hplBase;
			// i > j only between two blocks of one pose (a repeated pair), on its diagonal destination
			if (S.hplRowInd[i] != S.blkRow[k] || S.hplRowInd[j] != S.blkCol[k] || S.hplLm[S.prodI[n]] != S.hplLm[S.prodJ[n]] ||
				(i > j && S.blkRow[k] != S.blkCol[k]))
				return fail(CUBA_ERR_INVALID, "structure self-check: product list");
		}
	return CUBA_OK;
}

/* host side of the PCG setup on the CPU (no device needed): structure -> row partition over nCtas CTAs -> aggregates and coarse
 * lists with at most maxAgg aggregates; runs the invariants of check_pcg_partition.  info[8] = G, gs, A, needMax, maxRows,
 * blkMax, maxNeedAgg, size of the coarse lists. */
int cuba_debug_pcg_partition(const cuba_problem* p, int nCtas, int maxAgg, int32_t* info)
{
	if (!p || nCtas < 1 || maxAgg < 1) return fail(CUBA_ERR_INVALID, "pcg_partition: bad arguments");
	Structure S;
	const char* err = "";
	if (!build_structure(p->Pall, p->numP, p->Lall, p->numL, p->E2, p->idx2, p->E3, p->idx3, 0, 1, TILE, S, &err)) return fail(CUBA_ERR_INVALID, err);
	if (S.numP < 1) return fail(CUBA_ERR_INVALID, "pcg_partition: no free pose");
	const int G = std::max(1, std::min(nCtas, S.numP));
	PcgPartition P; CoarsePartition C;
	build_pcg_partition(S.numP, S.nfull, S.fRowPtr, S.fColInd, G, P);
	build_coarse_partition(S.numP, P, maxAgg, C);
	build_coarse_lists(S.numP, S.nfull, S.fRowPtr, S.fColInd, C);
	const char* bad = check_pcg_partition(S.numP, S.nfull, S.fRowPtr, S.fColInd, P, C);
	if (bad) return fail(CUBA_ERR_INVALID, std::string("pcg_partition self-check: ") + bad);
	if (info) {
		info[0] = P.G; info[1] = C.gs; info[2] = C.A; info[3] = P.needMax; info[4] = P.maxRows; info[5] = P.blkMax; info[6] = C.maxNeedAgg; info[7] = (int32_t)C.cbList.size();
		info[8] = (int32_t)pcg3_fixed_bytes(P.needMax, P.maxRows, sizeof(double));
	}
	return CUBA_OK;
}

/* host side of the row-distributed PCG plan on the CPU (no device needed): info[8] = ok, G, gs, A, needMax, maxRows, maxNeedAgg,
 * number of rows some other rank needs (halo rows) */
int cuba_debug_pcg5_plan(const cuba_problem* p, int world, int numSMs, int maxAgg, int32_t* info)
{
	return cuba_debug_pcg5_plan_apc(p, world, numSMs, maxAgg, 1, info, nullptr);
}

int cuba_debug_pcg5_plan_apc(const cuba_problem* p, int world, int numSMs, int maxAgg, int aggsPerCta, int32_t* info, uint64_t* hash)
{
	if (!p || world < 1 || world > 8 || numSMs < 1 || maxAgg < 1 || aggsPerCta < 1 || aggsPerCta > 3) return fail(CUBA_ERR_INVALID, "pcg5_plan: bad arguments");
	Structure S;
	const char* err = "";
	if (!build_structure(p->Pall, p->numP, p->Lall, p->numL, p->E2, p->idx2, p->E3, p->idx3, 0, 1, TILE, S, &err)) return fail(CUBA_ERR_INVALID, err);
	Pcg5Plan plan;
	build_pcg5_plan(S.numP, S.nfull, S.fRowPtr, S.fColInd, world, numSMs, maxAgg, 2 * PCG5_BLOCK / 6, plan, nullptr, aggsPerCta);
	if (info) for (int i = 0; i < 11; i++) info[i] = 0;
	if (hash) *hash = 0;
	if (!plan.ok) return CUBA_OK;
	const char* bad = check_pcg5_plan(S.numP, S.nfull, S.fRowPtr, S.fColInd, plan);
	if (bad) return fail(CUBA_ERR_INVALID, std::string("pcg5_plan self-check: ") + bad);
	if (info) {
		int halo = 0;
		for (unsigned char m : plan.rowPeers) if (m) halo++;
		info[0] = 1; info[1] = plan.G; info[2] = plan.gs; info[3] = plan.A; info[4] = plan.P.needMax; info[5] = plan.P.maxRows; info[6] = plan.C.maxNeedAgg; info[7] = halo;
		info[8] = plan.P.blkMax;
		// the two launch shapes' layouts as setup_pcg5 sizes them (the staging does not depend on the cached-block count)
		p5t::Pcg5Dims t{};
		t.needMax = plan.P.needMax; t.maxRows = plan.P.maxRows; t.ccCap = p5t::pcg5t_cc_cap(plan.P.blkMax);
		Pcg5Dims d{};
		d.needMax = plan.P.needMax; d.maxRows = plan.P.maxRows;
		info[9] = w_staging_columns(p5t::Pcg5Layout<double>(t));
		info[10] = w_staging_columns(Pcg5Layout<double>(d));
	}
	if (hash) {
		uint64_t h = 1469598103934665603ull;
		auto mix = [&h](const void* data, size_t bytes) {
			const unsigned char* b = (const unsigned char*)data;
			for (size_t i = 0; i < bytes; i++) { h ^= b[i]; h *= 1099511628211ull; }
		};
		auto vec = [&mix](const std::vector<int>& v) { const uint64_t n = v.size(); mix(&n, sizeof n); mix(v.data(), v.size() * sizeof(int)); };
		const int scal[] = { plan.G, plan.gs, plan.A, plan.P.needMax, plan.P.blkMax, plan.P.maxRows, plan.C.maxNeedAgg };
		mix(scal, sizeof scal);
		for (const std::vector<int>* v : { &plan.P.rows, &plan.P.nptr, &plan.P.ncol, &plan.P.local, &plan.C.aggRow, &plan.C.rowAgg, &plan.C.naPtr,
			&plan.C.naList, &plan.C.needAgg, &plan.C.rowOf, &plan.C.cbPtr, &plan.C.cbList }) vec(*v);
		mix(plan.rowPeers.data(), plan.rowPeers.size());
		*hash = h;
	}
	return CUBA_OK;
}

int cuba_debug_pcg5t_layout(const cuba_problem* p, int numSMs, int aggsPerCtaTop, int scalarBytes, int64_t smemBudget, int32_t* info)
{
	if (!p || numSMs < 1 || aggsPerCtaTop < 1 || aggsPerCtaTop > 3 || (scalarBytes != 4 && scalarBytes != 8) || smemBudget < 0 || !info)
		return fail(CUBA_ERR_INVALID, "pcg5t_layout: bad arguments");
	Structure S;
	const char* err = "";
	if (!build_structure(p->Pall, p->numP, p->Lall, p->numL, p->E2, p->idx2, p->E3, p->idx3, 0, 1, TILE, S, &err)) return fail(CUBA_ERR_INVALID, err);
	for (int i = 0; i < 12; i++) info[i] = 0;
	for (int apc = aggsPerCtaTop; apc >= 1; apc--) {
		Pcg5Plan plan;
		build_pcg5_plan(S.numP, S.nfull, S.fRowPtr, S.fColInd, 1, numSMs, PCG5_MAXAGG, 2 * PCG5_BLOCK / 6, plan, nullptr, apc);
		if (!plan.ok || plan.P.maxRows * 6 > p5t::Pcg5Shape::BLOCK) continue;
		p5t::Pcg5Dims t = pcg5t_plan_dims(plan);
		auto report = [&](auto lay) {
			const int cached = std::max(plan.P.blkMax - p5t::Pcg5Shape::REGBLK, 0);
			const size_t vals[12] = { 1, (size_t)apc, (size_t)t.capBlocks, (size_t)(cached - t.capBlocks), (size_t)t.zhInSmem, lay.total,
				lay.r - lay.blk, lay.p - lay.r, lay.rc - lay.cc, lay.c - lay.rc, lay.ls - lay.zh, lay.loc - lay.ai };
			for (int i = 0; i < 12; i++) info[i] = (int32_t)vals[i];
		};
		if (scalarBytes == 8) { if (!p5t::pcg5t_fit<double>(t, plan.P.blkMax, apc, (size_t)smemBudget)) continue; report(p5t::Pcg5Layout<double>(t)); }
		else { if (!p5t::pcg5t_fit<float>(t, plan.P.blkMax, apc, (size_t)smemBudget)) continue; report(p5t::Pcg5Layout<float>(t)); }
		break;
	}
	return CUBA_OK;
}

int cuba_debug_dense_layout(const cuba_problem* p, int32_t* info, int32_t* map)
{
	if (!p) return fail(CUBA_ERR_INVALID, "dense_layout: null problem");
	if (p->numP > dchol::MAX_POSES && p->numL > 0) return dense_cap_error(p->numP);
	Structure S;
	const char* err = "";
	if (!build_structure(p->Pall, p->numP, p->Lall, p->numL, p->E2, p->idx2, p->E3, p->idx3, 0, 1, TILE, S, &err)) return fail(CUBA_ERR_INVALID, err);
	const int n = 6 * S.numP, nt = dchol::tile_rows(n);
	std::vector<int> m;
	build_dense_block_map(S.numP, S.fRowPtr, S.fColInd, m);
	if (info) {
		const int64_t v[5] = { S.numP, n, nt, (int64_t)cdense::tiles(nt), (int64_t)(dchol::tile_doubles(n) * sizeof(double) >> 20) };
		for (int i = 0; i < 5; i++) info[i] = (int32_t)v[i];
	}
	if (map && !m.empty()) memcpy(map, m.data(), sizeof(int) * m.size());
	return CUBA_OK;
}

int cuba_bench_stage(cuba_engine* e, int stage, int reps, int flush, double lambda, double* ms) { ENGINE_OR_FAIL(e); return e->impl->bench_stage(stage, reps, flush, lambda, ms); }

}  // extern "C"
