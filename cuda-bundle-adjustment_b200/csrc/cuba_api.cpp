// cuba_api.cpp -- cuba::CudaBundleAdjustment on top of the C ABI (include/cuba_b200.h).
//
// Host-side mirror of the reference's graph container + initialize():
//   graph container      reference src/cuda_bundle_adjustment.cpp:677-781
//   index assignment     cpp:142-200  (ascending id, free first, fixed appended, edge-less vertices skipped)
//   edge flattening      cpp:202-243  (monocular ids first, then stereo; both-fixed edges dropped)
//   finalize/getChiSqs   cpp:512-543  (write-back of q,t,Xw into the caller's vertices, per-edge chi2)
// Differences, on purpose:
//   * edges are kept in insertion order (the reference iterates an unordered_set, so its order depends on heap addresses);
//   * the per-pose cameras are rebuilt on every initialize() (the reference never clears cameras_);
//   * removing a vertex copies its edge set before erasing from it;
//   * initialize() is built for repeated local-BA calls: vertices are looked up through hash maps and walked in a cached
//     ascending-id order (re-sorted only after an add/remove), removals are O(1) tombstones compacted at the next initialize(),
//     the flat arrays live in page-locked memory (the engine's H2D copies are plain DMA) and the edge pass is split over a few
//     host threads; the pointer -> chi2 map the reference rebuilds in every optimize() (cpp:541-542) is built on the first
//     chiSquared() call instead.
// Edge levels (include/cuba_b200_levels.h, which the reference does not have): one byte per list slot beside mono_ / stereo_, so that
// compaction, the dropping of both-fixed edges and the value-only initialize() carry them; a flat copy in the order of the flat
// arrays goes to the engine after set_problem only when some level is set; classifyEdges() decisions are fetched lazily.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/cuba_b200.h"
#include "../../include/cuda_bundle_adjustment.h"
#include "../../include/cuba_b200_levels.h"
#include "../../include/cuba_b200_pose.h"
#include "../../include/cuba_b200_points.h"
#include "../../include/cuba_b200_sim3.h"
#include "../../include/cuba_b200_solver.h"

namespace cuba
{

namespace
{

// grow-only host array in page-locked memory (pageable when no CUDA device is usable: initialize() itself needs no GPU)
template <typename T>
class HostBuf
{
public:
	HostBuf() {}
	HostBuf(const HostBuf&) = delete;
	HostBuf& operator=(const HostBuf&) = delete;
	~HostBuf() { release(); }
	void resize(size_t n)
	{
		if (n > cap_) {
			release();
			cap_ = n + n / 8 + 16;
			void* q = nullptr;
			if (cudaMallocHost(&q, cap_ * sizeof(T)) == cudaSuccess) { p_ = static_cast<T*>(q); pinned_ = true; }
			else { cudaGetLastError(); p_ = static_cast<T*>(std::malloc(cap_ * sizeof(T))); pinned_ = false; if (!p_) throw std::bad_alloc(); }
		}
		n_ = n;
	}
	T* data() { return p_; }
	const T* data() const { return p_; }
	size_t size() const { return n_; }
	T& operator[](size_t i) { return p_[i]; }
	const T& operator[](size_t i) const { return p_[i]; }
private:
	void release()
	{
		if (p_) { if (pinned_) cudaFreeHost(p_); else std::free(p_); }
		p_ = nullptr; cap_ = 0; n_ = 0;
	}
	T* p_ = nullptr; size_t n_ = 0, cap_ = 0; bool pinned_ = false;
};

// Host loops over vertex / edge objects are pointer chasing (memory-latency bound): a few threads, each prefetching ahead.
static unsigned host_threads(size_t n, size_t grain)
{
	const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
	return static_cast<unsigned>(std::max<size_t>(1, std::min<size_t>(std::min<size_t>(16, hw), n / grain + 1)));
}

// runs fn(t, begin, end) for the t-th of nthreads equal slices of [0, n)
template <class F>
static void parallel_slices(size_t n, unsigned nthreads, F fn)
{
	if (nthreads <= 1) { fn(0u, size_t(0), n); return; }
	std::vector<std::thread> pool;
	for (unsigned t = 1; t < nthreads; t++) pool.emplace_back(fn, t, n * t / nthreads, n * (t + 1) / nthreads);
	fn(0u, size_t(0), n / nthreads);
	for (auto& th : pool) th.join();
}

template <class F>
static void parallel_for(size_t n, F fn)
{
	parallel_slices(n, host_threads(n, 32768), [&fn](unsigned, size_t b, size_t e) { fn(b, e); });
}

class Impl : public CudaBundleAdjustment
{
public:
	Impl()
	{
		kernels_[0] = { 0, 0.0 };
		kernels_[1] = { 0, 0.0 };
	}
	~Impl() override { if (engine_) cuba_engine_destroy(engine_); }

	void addPoseVertex(PoseVertex* v) override { if (poses_.insert({ v->id, v }).second) orderDirty_ = true; }
	void addLandmarkVertex(LandmarkVertex* v) override { if (landmarks_.insert({ v->id, v }).second) orderDirty_ = true; }

	void addMonocularEdge(MonoEdge* e) override
	{
		if (!member_.insert(e).second) return;
		edgeVersion_++;
		mono_.push_back(e); levMono_.push_back(0);
		slotValid_ = false;
		e->vertexP->edges.insert(e); e->vertexL->edges.insert(e);
	}
	void addStereoEdge(StereoEdge* e) override
	{
		if (!member_.insert(e).second) return;
		edgeVersion_++;
		stereo_.push_back(e); levStereo_.push_back(0);
		slotValid_ = false;
		e->vertexP->edges.insert(e); e->vertexL->edges.insert(e);
	}

	PoseVertex* poseVertex(int id) const override { return poses_.at(id); }
	LandmarkVertex* landmarkVertex(int id) const override { return landmarks_.at(id); }

	void removePoseVertex(PoseVertex* v) override
	{
		auto it = poses_.find(v->id);
		if (it == poses_.end()) return;
		const std::vector<BaseEdge*> es(it->second->edges.begin(), it->second->edges.end());
		for (auto e : es) removeEdge(e);
		poses_.erase(it);
		orderDirty_ = true;
	}
	void removeLandmarkVertex(LandmarkVertex* v) override
	{
		auto it = landmarks_.find(v->id);
		if (it == landmarks_.end()) return;
		const std::vector<BaseEdge*> es(it->second->edges.begin(), it->second->edges.end());
		for (auto e : es) removeEdge(e);
		landmarks_.erase(it);
		orderDirty_ = true;
	}
	// O(1): the slot in the insertion-ordered list becomes a tombstone, dropped by the next initialize()
	void removeEdge(BaseEdge* e) override
	{
		if (auto p = e->poseVertex()) p->edges.erase(e);
		if (auto l = e->landmarkVertex()) l->edges.erase(e);
		if (!member_.erase(e)) return;
		edgeVersion_++;
		tombstones_[e]++;
		(e->dim() == 2 ? deadMono_ : deadStereo_)++;
	}

	size_t nposes() const override { return poses_.size(); }
	size_t nlandmarks() const override { return landmarks_.size(); }
	size_t nedges() const override { return mono_.size() + stereo_.size() - deadMono_ - deadStereo_; }

	void setRobustKernels(RobustKernelType kernelType, double delta, EdgeType edgeType) override
	{
		kernels_[static_cast<int>(edgeType)] = { static_cast<int>(kernelType), delta };
	}

	void initialize() override
	{
		const auto t0 = std::chrono::steady_clock::now();
		levelsFromDevice();      // classifyEdges() decisions into the lists while their slots still match the uploaded problem
		compactEdges();
		if (orderDirty_) {
			orderP_.clear(); orderL_.clear();
			orderP_.reserve(poses_.size()); orderL_.reserve(landmarks_.size());
			for (const auto& kv : poses_) orderP_.push_back(kv.second);
			for (const auto& kv : landmarks_) orderL_.push_back(kv.second);
			std::sort(orderP_.begin(), orderP_.end(), [](const PoseVertex* a, const PoseVertex* b) { return a->id < b->id; });
			std::sort(orderL_.begin(), orderL_.end(), [](const LandmarkVertex* a, const LandmarkVertex* b) { return a->id < b->id; });
			orderDirty_ = false;
		}
		// index assignment: ascending id, free vertices first, fixed ones appended, vertices without edges skipped
		// (if neither the numbering nor the edge lists moved since the last initialize(), the edge pass below only refreshes values)
		prevP_.swap(vP_);
		const int prevNumP = numP_, prevNumL = numL_;
		vP_.clear();
		vP_.reserve(orderP_.size());
		size_t nFixedP = 0, nFixedL = 0;
		for (PoseVertex* v : orderP_) { if (v->edges.empty()) continue; if (v->fixed) nFixedP++; else { v->iP = static_cast<int>(vP_.size()); vP_.push_back(v); } }
		numP_ = static_cast<int>(vP_.size());
		if (nFixedP) for (PoseVertex* v : orderP_) if (v->fixed && !v->edges.empty()) { v->iP = static_cast<int>(vP_.size()); vP_.push_back(v); }
		// landmarks (many): pass 1 classifies every vertex (0 = no edges, 1 = free, 2 = fixed) and counts per slice, pass 2 writes
		// index, list entry and coordinates at the slice's offsets -- same numbering as a serial walk in ascending id
		{
			const size_t nl = orderL_.size();
			const unsigned nt = host_threads(nl, 16384);
			cls_.resize(nl);
			std::vector<size_t> cntFree(nt + 1, 0), cntFixed(nt + 1, 0);
			parallel_slices(nl, nt, [&](unsigned tix, size_t b, size_t e) {
				size_t nf = 0, nx = 0;
				for (size_t i = b; i < e; i++) {
					if (i + 8 < e) __builtin_prefetch(orderL_[i + 8]);
					const LandmarkVertex* v = orderL_[i];
					const unsigned char c = v->edges.empty() ? 0 : (v->fixed ? 2 : 1);
					cls_[i] = c; nf += c == 1; nx += c == 2;
				}
				cntFree[tix + 1] = nf; cntFixed[tix + 1] = nx;
			});
			for (unsigned t = 0; t < nt; t++) { cntFree[t + 1] += cntFree[t]; cntFixed[t + 1] += cntFixed[t]; }
			numL_ = static_cast<int>(cntFree[nt]);
			nFixedL = cntFixed[nt];
			sameNumbering_ = vL_.size() == cntFree[nt] + cntFixed[nt] && numL_ == prevNumL;
			vL_.resize(cntFree[nt] + cntFixed[nt]);
			Xw_.resize(3 * vL_.size());
			std::vector<unsigned char> moved(nt, 0);
			parallel_slices(nl, nt, [&](unsigned tix, size_t b, size_t e) {
				size_t wf = cntFree[tix], wx = cntFree[nt] + cntFixed[tix];
				unsigned char mv = 0;
				for (size_t i = b; i < e; i++) {
					if (i + 8 < e) __builtin_prefetch(orderL_[i + 8], 1);
					if (!cls_[i]) continue;
					LandmarkVertex* v = orderL_[i];
					const size_t w = cls_[i] == 1 ? wf++ : wx++;
					mv |= vL_[w] != v;
					v->iL = static_cast<int>(w); vL_[w] = v;
					for (int k = 0; k < 3; k++) Xw_[3 * w + k] = v->Xw.data()[k];
				}
				moved[tix] = mv;
			});
			for (unsigned char mv : moved) if (mv) sameNumbering_ = false;
		}
		sameNumbering_ = sameNumbering_ && numP_ == prevNumP && vP_ == prevP_;

		q_.resize(4 * vP_.size()); t_.resize(3 * vP_.size()); cam_.resize(5 * vP_.size());
		for (size_t i = 0; i < vP_.size(); i++) {
			const PoseVertex* v = vP_[i];
			for (int k = 0; k < 4; k++) q_[4 * i + k] = v->q.coeffs().data()[k];
			for (int k = 0; k < 3; k++) t_[3 * i + k] = v->t.data()[k];
			cam_[5 * i] = v->camera.fx; cam_[5 * i + 1] = v->camera.fy; cam_[5 * i + 2] = v->camera.cx;
			cam_[5 * i + 3] = v->camera.cy; cam_[5 * i + 4] = v->camera.bf;
		}

		// edges: every list entry is written at its own position by a few threads; only if an edge with both ends fixed
		// turned up (they are dropped, cpp:210-211) the arrays are closed up afterwards
		idx2_.resize(2 * mono_.size()); meas2_.resize(2 * mono_.size()); om2_.resize(mono_.size());
		idx3_.resize(2 * stereo_.size()); meas3_.resize(3 * stereo_.size()); om3_.resize(stereo_.size());
		const size_t n2 = mono_.size(), n3 = stereo_.size(), total = n2 + n3;
		lev_.resize(total);
		levFlatStale_ = false;
		const unsigned nthreads = host_threads(total, 65536);
		if (flatValid_ && sameNumbering_ && flatVersion_ == edgeVersion_ && om2_.size() == n2 && om3_.size() == n3) {
			// same edges in the same order between the same indices, none dropped: the index pairs and the position -> edge lists of
			// the last initialize() still hold; the caller may have edited measurements / information in place
			parallel_slices(total, nthreads, [&](unsigned, size_t b, size_t e) {
				for (size_t k = b; k < e; k++) {
					if (k + 16 < e) __builtin_prefetch(k + 16 < n2 ? static_cast<const void*>(mono_[k + 16]) : static_cast<const void*>(stereo_[k + 16 - n2]));
					if (k < n2) {
						const MonoEdge* ed = mono_[k];
						meas2_[2 * k] = ed->measurement.data()[0]; meas2_[2 * k + 1] = ed->measurement.data()[1];
						om2_[k] = ed->information;
						lev_[k] = levMono_[k];
					} else {
						const size_t j = k - n2;
						const StereoEdge* ed = stereo_[j];
						for (int c = 0; c < 3; c++) meas3_[3 * j + c] = ed->measurement.data()[c];
						om3_[j] = ed->information;
						lev_[k] = levStereo_[j];
					}
				}
			});
			stats_.clear();
			uploaded_ = false;
			initSeconds_ = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
			initialized_ = true;
			return;
		}
		auto am = takeList(mono_.size());
		auto as = takeList(stereo_.size());
		std::vector<size_t> dropped(nthreads, 0);
		parallel_slices(total, nthreads, [&](unsigned tix, size_t b, size_t e) {
			// two prefetch distances: the edge object 16 ahead, its landmark (read through the edge) 8 ahead
			auto edgeAt = [&](size_t k) -> const BaseEdge* { return k < n2 ? static_cast<const BaseEdge*>(mono_[k]) : static_cast<const BaseEdge*>(stereo_[k - n2]); };
			size_t drop = 0;
			for (size_t k = b; k < e; k++) {
				if (k + 16 < e) __builtin_prefetch(edgeAt(k + 16));
				if (k + 8 < e) __builtin_prefetch(k + 8 < n2 ? static_cast<const void*>(mono_[k + 8]->vertexL) : static_cast<const void*>(stereo_[k + 8 - n2]->vertexL));
				if (k < n2) {
					const MonoEdge* ed = mono_[k];
					const PoseVertex* vp = ed->vertexP; const LandmarkVertex* vl = ed->vertexL;
					if (vp->fixed && vl->fixed) drop++;
					(*am)[k] = ed;
					idx2_[2 * k] = vp->iP; idx2_[2 * k + 1] = vl->iL;
					meas2_[2 * k] = ed->measurement.data()[0]; meas2_[2 * k + 1] = ed->measurement.data()[1];
					om2_[k] = ed->information;
					lev_[k] = levMono_[k];
				} else {
					const size_t j = k - n2;
					const StereoEdge* ed = stereo_[j];
					const PoseVertex* vp = ed->vertexP; const LandmarkVertex* vl = ed->vertexL;
					if (vp->fixed && vl->fixed) drop++;
					(*as)[j] = ed;
					idx3_[2 * j] = vp->iP; idx3_[2 * j + 1] = vl->iL;
					for (int c = 0; c < 3; c++) meas3_[3 * j + c] = ed->measurement.data()[c];
					om3_[j] = ed->information;
					lev_[k] = levStereo_[j];
				}
			}
			dropped[tix] = drop;
		});
		size_t ndrop = 0;
		for (size_t d : dropped) ndrop += d;
		flatMono_.clear(); flatStereo_.clear();
		if (ndrop) {
			// (the levels close up in place: the stereo levels start behind the kept monocular ones)
			size_t w = 0;
			for (size_t k = 0; k < n2; k++) {
				const MonoEdge* ed = mono_[k];
				if (ed->vertexP->fixed && ed->vertexL->fixed) continue;
				(*am)[w] = ed; idx2_[2 * w] = idx2_[2 * k]; idx2_[2 * w + 1] = idx2_[2 * k + 1];
				meas2_[2 * w] = meas2_[2 * k]; meas2_[2 * w + 1] = meas2_[2 * k + 1]; om2_[w] = om2_[k]; lev_[w] = lev_[k];
				flatMono_.push_back(k); w++;
			}
			am->resize(w); idx2_.resize(2 * w); meas2_.resize(2 * w); om2_.resize(w);
			const size_t w2 = w;
			w = 0;
			for (size_t j = 0; j < n3; j++) {
				const StereoEdge* ed = stereo_[j];
				if (ed->vertexP->fixed && ed->vertexL->fixed) continue;
				(*as)[w] = ed; idx3_[2 * w] = idx3_[2 * j]; idx3_[2 * w + 1] = idx3_[2 * j + 1];
				for (int c = 0; c < 3; c++) meas3_[3 * w + c] = meas3_[3 * j + c];
				om3_[w] = om3_[j]; lev_[w2 + w] = lev_[n2 + j];
				flatStereo_.push_back(j); w++;
			}
			as->resize(w); idx3_.resize(2 * w); meas3_.resize(3 * w); om3_.resize(w);
			lev_.resize(w2 + w);
		}
		activeMono_ = am; activeStereo_ = as;
		flatValid_ = ndrop == 0; flatVersion_ = edgeVersion_;
		stats_.clear();
		uploaded_ = false;
		initSeconds_ = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
		initialized_ = true;
	}

	void optimize(int niterations) override
	{
		if (!initialized_) initialize();
		ensureEngine();
		check(cuba_engine_set_robust_kernel(engine_, CUBA_EDGE_MONOCULAR, kernels_[0].type, kernels_[0].delta));
		check(cuba_engine_set_robust_kernel(engine_, CUBA_EDGE_STEREO, kernels_[1].type, kernels_[1].delta));
		if (!uploaded_ || solverChanged_) {
			// the reference builds its structure inside the first optimize() iteration (cpp:804-805); a new linear solver takes effect
			// through set_problem too, from the estimate of the last optimize() (the flat arrays hold it), keeping the levels
			if (uploaded_) levelsFromDevice();
			check(cuba_engine_set_linear_solver(engine_, solver_ == LinearSolverType::DENSE_CHOLESKY ? CUBA_SOLVER_DENSE_CHOLESKY : CUBA_SOLVER_PCG));
			cuba_problem p;
			flatProblem(p);
			check(cuba_engine_set_problem(engine_, &p));
			solverChanged_ = false;      // only once the engine holds the problem for the chosen solver: a refused upload is tried again
			uploaded_ = true;
			levDevNewer_ = false;
			// set_problem left every level at 0: lev_ must first take the levels set since initialize() before it is compared with that
			if (levFlatStale_) rebuildFlatLevels();
			levUploaded_ = std::none_of(lev_.data(), lev_.data() + lev_.size(), [](unsigned char l) { return l != 0; });
		}
		pushLevels();
		std::vector<cuba_iter_stat> st(niterations > 0 ? niterations : 1);
		int n = 0;
		if (niterations > 0) check(cuba_engine_optimize(engine_, niterations, st.data(), &n));
		// the reference appends to stats_ across optimize() calls (cleared by initialize()), cpp:848
		for (int i = 0; i < n; i++) stats_.push_back({ st[i].iteration, st[i].chi2 });

		// finalize(): write the estimate back into the caller's vertices (fixed ones too)
		check(cuba_engine_get_state(engine_, q_.data(), t_.data(), Xw_.data()));
		for (size_t i = 0; i < vP_.size(); i++) {
			for (int k = 0; k < 4; k++) vP_[i]->q.coeffs().data()[k] = q_[4 * i + k];
			for (int k = 0; k < 3; k++) vP_[i]->t.data()[k] = t_[3 * i + k];
		}
		parallel_for(vL_.size(), [this](size_t b, size_t e) { for (size_t i = b; i < e; i++) for (int k = 0; k < 3; k++) vL_[i]->Xw.data()[k] = Xw_[3 * i + k]; });

		// getChiSqs(): the values now, the pointer -> value map when somebody asks (chiSquared)
		chi_.resize(om2_.size() + om3_.size());
		if (chi_.size()) check(cuba_engine_get_chi2(engine_, chi_.data()));
		chiMono_ = activeMono_; chiStereo_ = activeStereo_;
		chiIndexValid_ = false;

		double sec[CUBA_PROF_NUM] = { 0 };
		check(cuba_engine_get_profile(engine_, sec));
		static const char* names[CUBA_PROF_NUM] = { "0: Initialize Optimizer", "1: Build Structure", "2: Compute Error",
			"3: Build System", "4: Schur Complement", "5: Symbolic Decomposition", "6: Numerical Decomposition", "7: Update Solution" };
		profile_.clear();
		for (int i = 0; i < CUBA_PROF_NUM; i++) profile_[names[i]] = sec[i];
		profile_[names[0]] += initSeconds_;
	}

	// the flat arrays of the last initialize() (also behind cuba_debug_dropin_problem)
	bool flatProblem(cuba_problem& p) const
	{
		if (!initialized_) return false;
		p.Pall = static_cast<int32_t>(vP_.size()); p.numP = numP_; p.Lall = static_cast<int32_t>(vL_.size()); p.numL = numL_;
		p.q = q_.data(); p.t = t_.data(); p.cam = cam_.data(); p.Xw = Xw_.data();
		p.E2 = static_cast<int32_t>(om2_.size()); p.idx2 = idx2_.data(); p.meas2 = meas2_.data(); p.omega2 = om2_.data();
		p.E3 = static_cast<int32_t>(om3_.size()); p.idx3 = idx3_.data(); p.meas3 = meas3_.data(); p.omega3 = om3_.data();
		return true;
	}

	// ---- linear solver (include/cuba_b200_solver.h) ----
	void setLinearSolver(LinearSolverType type)
	{
		if (type == solver_) return;
		solver_ = type;
		solverChanged_ = true;
	}
	LinearSolverType linearSolver() const { return solver_; }

	// ---- edge levels (include/cuba_b200_levels.h) ----
	void setEdgeLevel(BaseEdge* e, int level)
	{
		unsigned char& l = levelOf(e);
		const unsigned char v = level != 0;
		if (l == v) return;
		l = v;
		levFlatStale_ = true; levUploaded_ = false;
	}
	int edgeLevel(const BaseEdge* e) { return levelOf(e); }
	OutlierCounts classifyEdges(const OutlierTest& test)
	{
		if (!engine_ || !uploaded_) throw std::logic_error("cuba::classifyEdges: no optimize() since the last initialize()");
		pushLevels();
		int32_t c[4] = { 0, 0, 0, 0 };
		const int flags = (test.requirePositiveDepth ? CUBA_CLASSIFY_DEPTH : 0) | (test.reinclude ? CUBA_CLASSIFY_REINCLUDE : 0);
		check(cuba_engine_classify_edges(engine_, test.chi2Mono, test.chi2Stereo, flags, c));
		if (c[2] + c[3] > 0) levDevNewer_ = true;
		OutlierCounts out;
		out.includedMono = static_cast<size_t>(c[0]); out.includedStereo = static_cast<size_t>(c[1]);
		out.excluded = static_cast<size_t>(c[2]); out.reincluded = static_cast<size_t>(c[3]);
		return out;
	}
	// include/cuba_b200_points.h: the held problem's free landmarks (all of them, or `list`) refined in place on the engine
	std::vector<OutlierCounts> optimizeLandmarks(const std::vector<cuba_pose_round>& rounds, const std::vector<LandmarkVertex*>* list)
	{
		if (!engine_ || !uploaded_) throw std::logic_error("cuba::optimizeLandmarks: no optimize() since the last initialize()");
		std::vector<int32_t> idx;
		if (list) {
			idx.reserve(list->size());
			for (const LandmarkVertex* v : *list) {
				// a free landmark of the uploaded graph: its index names it in the flat problem
				if (!v || v->iL < 0 || v->iL >= numL_ || vL_[static_cast<size_t>(v->iL)] != v)
					throw std::invalid_argument("cuba::optimizeLandmarks: a vertex that is not a free landmark of the uploaded graph");
				idx.push_back(v->iL);
			}
		}
		pushLevels();
		const size_t R = rounds.size();
		std::vector<int32_t> c(4 * std::max<size_t>(R, 1), 0);
		const int32_t n = list ? static_cast<int32_t>(idx.size()) : numL_;
		const int rc = cuba_engine_optimize_landmarks(engine_, list ? idx.data() : nullptr, n, static_cast<int>(R), rounds.data(), c.data(),
			nullptr, nullptr);
		if (rc == CUBA_ERR_INVALID) throw std::invalid_argument(std::string("cuba::optimizeLandmarks: ") + cuba_last_error());
		check(rc);
		std::vector<OutlierCounts> out(R);
		for (size_t r = 0; r < R; r++) {
			out[r].includedMono = static_cast<size_t>(c[4 * r]); out[r].includedStereo = static_cast<size_t>(c[4 * r + 1]);
			out[r].excluded = static_cast<size_t>(c[4 * r + 2]); out[r].reincluded = static_cast<size_t>(c[4 * r + 3]);
			if (c[4 * r + 2] + c[4 * r + 3] > 0) levDevNewer_ = true;
		}
		// optimize()'s finalize for the refined vertices, and the per-edge chi2 it refreshes
		check(cuba_engine_get_state(engine_, q_.data(), t_.data(), Xw_.data()));
		auto put = [this](size_t i) { for (int k = 0; k < 3; k++) vL_[i]->Xw.data()[k] = Xw_[3 * i + k]; };
		if (list) for (int32_t i : idx) put(static_cast<size_t>(i));
		else parallel_for(static_cast<size_t>(numL_), [&](size_t b, size_t e) { for (size_t i = b; i < e; i++) put(i); });
		chi_.resize(om2_.size() + om3_.size());
		if (chi_.size()) check(cuba_engine_get_chi2(engine_, chi_.data()));
		chiMono_ = activeMono_; chiStereo_ = activeStereo_;
		chiIndexValid_ = false;
		return out;
	}
	// the engine optimizePoses() runs on (include/cuba_b200_pose.h): this object's, created on demand
	cuba_engine* poseEngine()
	{
		ensureEngine();
		return engine_;
	}
	// the flat levels with every level set so far applied (also behind cuba_debug_dropin_levels)
	bool flatLevels(const uint8_t** p, int32_t* n)
	{
		if (!initialized_) return false;
		levelsFromDevice();
		if (levFlatStale_) rebuildFlatLevels();
		if (p) *p = lev_.data();
		if (n) *n = static_cast<int32_t>(lev_.size());
		return true;
	}

	void clear() override
	{
		levMono_.clear(); levStereo_.clear(); slot_.clear(); slotValid_ = false;
		flatMono_.clear(); flatStereo_.clear(); lev_.resize(0);
		levFlatStale_ = false; levUploaded_ = true; levDevNewer_ = false;
		poses_.clear(); landmarks_.clear(); mono_.clear(); stereo_.clear(); member_.clear(); tombstones_.clear();
		deadMono_ = deadStereo_ = 0; orderDirty_ = true;
		edgeVersion_++; flatValid_ = false;
		stats_.clear(); initialized_ = false; uploaded_ = false;
	}

	const BatchStatistics& batchStatistics() const override { return stats_; }
	const TimeProfile& timeProfile() const override { return profile_; }
	double chiSquared(const BaseEdge* e) const override
	{
		if (!chiIndexValid_) {
			chiIndex_.clear();
			const size_t n2 = chiMono_ ? chiMono_->size() : 0, n3 = chiStereo_ ? chiStereo_->size() : 0;
			chiIndex_.reserve(n2 + n3);
			for (size_t i = 0; i < n2; i++) chiIndex_[(*chiMono_)[i]] = i;
			for (size_t i = 0; i < n3; i++) chiIndex_[(*chiStereo_)[i]] = n2 + i;
			chiIndexValid_ = true;
		}
		auto it = chiIndex_.find(e);
		return it == chiIndex_.end() || it->second >= chi_.size() ? 0.0 : chi_[it->second];
	}

private:
	struct Kernel { int type; double delta; };

	// drops the tombstoned slots (earliest occurrences first: an edge removed and added again keeps its new position)
	void compactEdges()
	{
		if (tombstones_.empty()) return;
		auto sweep = [this](auto& vec, std::vector<unsigned char>& lev) {
			size_t w = 0;
			for (size_t k = 0; k < vec.size(); k++) {
				auto it = tombstones_.find(vec[k]);
				if (it != tombstones_.end()) { if (--it->second == 0) tombstones_.erase(it); continue; }
				lev[w] = lev[k];
				vec[w++] = vec[k];
			}
			vec.resize(w); lev.resize(w);
		};
		sweep(mono_, levMono_); sweep(stereo_, levStereo_);
		tombstones_.clear();
		deadMono_ = deadStereo_ = 0;
		slotValid_ = false;
	}

	// the level of the list slot that holds e now (the last one: an edge removed and added again has a new slot)
	unsigned char& levelOf(const BaseEdge* e)
	{
		if (!member_.count(e)) throw std::out_of_range("cuba: the optimizer does not hold this edge");
		levelsFromDevice();
		if (!slotValid_) {
			slot_.clear();
			slot_.reserve(mono_.size() + stereo_.size());
			for (size_t k = 0; k < mono_.size(); k++) slot_[mono_[k]] = k;
			for (size_t k = 0; k < stereo_.size(); k++) slot_[stereo_[k]] = k;
			slotValid_ = true;
		}
		const size_t k = slot_.at(e);
		return e->dim() == 2 ? levMono_[k] : levStereo_[k];
	}
	// list slot of the w-th flat edge of the last initialize() (the identity unless it dropped edges with both ends fixed)
	size_t monoSlot(size_t w) const { return flatMono_.empty() ? w : flatMono_[w]; }
	size_t stereoSlot(size_t w) const { return flatStereo_.empty() ? w : flatStereo_[w]; }
	void rebuildFlatLevels()
	{
		const size_t n2 = om2_.size(), n3 = om3_.size();
		for (size_t w = 0; w < n2; w++) lev_[w] = levMono_[monoSlot(w)];
		for (size_t w = 0; w < n3; w++) lev_[n2 + w] = levStereo_[stereoSlot(w)];
		levFlatStale_ = false;
	}
	// classifyEdges() changed levels on the device: fetch them into the flat array and the lists (slots are stable until compaction)
	void levelsFromDevice()
	{
		if (!levDevNewer_) return;
		check(cuba_engine_get_edge_levels(engine_, lev_.data()));
		const size_t n2 = om2_.size(), n3 = om3_.size();
		for (size_t w = 0; w < n2; w++) levMono_[monoSlot(w)] = lev_[w];
		for (size_t w = 0; w < n3; w++) levStereo_[stereoSlot(w)] = lev_[n2 + w];
		levDevNewer_ = false;
	}
	// the levels set since the last upload to the engine (nothing when none changed)
	void pushLevels()
	{
		if (levFlatStale_) rebuildFlatLevels();
		if (levUploaded_) return;
		check(cuba_engine_set_edge_levels(engine_, lev_.data()));
		levUploaded_ = true;
	}

	// a position -> edge list for chiSquared(): the previous optimize()'s lists stay alive in chiMono_/chiStereo_, so the
	// lists rotate through a small pool instead of being allocated (and page-faulted in) on every initialize()
	std::shared_ptr<std::vector<const BaseEdge*>> takeList(size_t n)
	{
		for (auto& l : listPool_)
			if (l.use_count() == 1) { l->resize(n); return l; }
		listPool_.push_back(std::make_shared<std::vector<const BaseEdge*>>(n));
		return listPool_.back();
	}

	void ensureEngine()
	{
		if (engine_) return;
		cuba_config cfg{};
		cfg.device = -1; cfg.deterministic = 1;
#ifdef USE_FLOAT32
		cfg.use_fp32 = 1;
#endif
		check(cuba_engine_create(&cfg, &engine_));
	}
	static void check(int rc)
	{
		// the reference prints CUDA errors and continues (src/macro.h:22-27); failing loudly is safer
		if (rc != CUBA_OK) throw std::runtime_error(std::string("cuba_b200: ") + cuba_last_error());
	}

	std::unordered_map<int, PoseVertex*> poses_;
	std::unordered_map<int, LandmarkVertex*> landmarks_;
	std::vector<PoseVertex*> orderP_;          // ascending id, valid while !orderDirty_
	std::vector<LandmarkVertex*> orderL_;
	bool orderDirty_ = true;
	std::vector<MonoEdge*> mono_;              // insertion order, may hold tombstoned slots until the next initialize()
	std::vector<StereoEdge*> stereo_;
	// edge levels: one byte per list slot (compaction, dropped both-fixed edges and the value-only initialize() carry them)
	std::vector<unsigned char> levMono_, levStereo_;
	std::unordered_map<const BaseEdge*, size_t> slot_;   // edge -> its live slot, rebuilt after an add or a compaction
	bool slotValid_ = false;
	std::vector<size_t> flatMono_, flatStereo_;          // list slot of every flat edge when the last initialize() dropped edges
	bool levFlatStale_ = false;   // a level changed since lev_ was built
	bool levUploaded_ = true;     // the engine holds lev_ (a graph that never uses levels never uploads any)
	bool levDevNewer_ = false;    // classifyEdges() changed levels on the engine that lev_ and the lists do not have yet
	std::unordered_set<const BaseEdge*> member_;
	std::unordered_map<const BaseEdge*, int> tombstones_;
	size_t deadMono_ = 0, deadStereo_ = 0;
	Kernel kernels_[2];

	std::vector<PoseVertex*> vP_, prevP_;
	std::vector<LandmarkVertex*> vL_;
	size_t edgeVersion_ = 0, flatVersion_ = 0;   // edits of the edge lists / the version the flat edge arrays were built from
	bool flatValid_ = false, sameNumbering_ = false;
	std::shared_ptr<const std::vector<const BaseEdge*>> activeMono_, activeStereo_, chiMono_, chiStereo_;
	std::vector<std::shared_ptr<std::vector<const BaseEdge*>>> listPool_;
	std::vector<unsigned char> cls_;
	int numP_ = 0, numL_ = 0;
	HostBuf<double> q_, t_, cam_, Xw_, meas2_, om2_, meas3_, om3_, chi_;
	HostBuf<int32_t> idx2_, idx3_;
	HostBuf<unsigned char> lev_;                 // flat levels, order of the flat edge arrays
	bool initialized_ = false, uploaded_ = false;
	LinearSolverType solver_ = LinearSolverType::PCG;
	bool solverChanged_ = false;   // the engine holds the problem for the other solver: the next optimize() uploads it again
	double initSeconds_ = 0;

	cuba_engine* engine_ = nullptr;
	BatchStatistics stats_;
	TimeProfile profile_;
	mutable std::unordered_map<const BaseEdge*, size_t> chiIndex_;
	mutable bool chiIndexValid_ = false;
};

} // namespace

CudaBundleAdjustment::Ptr CudaBundleAdjustment::create() { return Ptr(new Impl()); }

// include/cuba_b200.h: cuba_debug_dropin_problem
static bool dropin_problem(CudaBundleAdjustment* obj, cuba_problem* out)
{
	const Impl* impl = dynamic_cast<const Impl*>(obj);
	return impl && out && impl->flatProblem(*out);
}
CudaBundleAdjustment::~CudaBundleAdjustment() {}

// include/cuba_b200_levels.h: free functions, so that the class keeps the reference's vtable
static Impl& impl_of(const CudaBundleAdjustment& ba)
{
	const Impl* impl = dynamic_cast<const Impl*>(&ba);
	if (!impl) throw std::invalid_argument("cuba: edge levels need an optimizer made by cuba::CudaBundleAdjustment::create()");
	return const_cast<Impl&>(*impl);      // reading a level may first fetch the device's decisions into the host lists
}
void setEdgeLevel(CudaBundleAdjustment& ba, BaseEdge* e, int level) { impl_of(ba).setEdgeLevel(e, level); }
int edgeLevel(const CudaBundleAdjustment& ba, const BaseEdge* e) { return impl_of(ba).edgeLevel(e); }
OutlierCounts classifyEdges(CudaBundleAdjustment& ba, const OutlierTest& test) { return impl_of(ba).classifyEdges(test); }

// include/cuba_b200_solver.h
void setLinearSolver(CudaBundleAdjustment& ba, LinearSolverType type) { impl_of(ba).setLinearSolver(type); }
LinearSolverType linearSolver(const CudaBundleAdjustment& ba) { return impl_of(ba).linearSolver(); }

// include/cuba_b200_pose.h
std::vector<PoseRound> orbSlam2PoseSchedule()
{
	std::vector<PoseRound> s(4);
	for (size_t r = 0; r < s.size(); r++) {
		if (r < 2) {
			s[r].kernelMono = s[r].kernelStereo = RobustKernelType::HUBER;
			s[r].deltaMono = std::sqrt(5.991); s[r].deltaStereo = std::sqrt(7.815);
		}
		s[r].test.chi2Mono = 5.991; s[r].test.chi2Stereo = 7.815;
		s[r].test.requirePositiveDepth = false; s[r].test.reinclude = true;
	}
	return s;
}

// the C ABI's rounds of a drop-in schedule; perProblem = the stat slots of one problem
static std::vector<cuba_pose_round> c_rounds(const std::vector<PoseRound>& schedule, size_t& perProblem)
{
	std::vector<cuba_pose_round> rounds(schedule.size());
	perProblem = 0;
	for (size_t r = 0; r < schedule.size(); r++) {
		const PoseRound& s = schedule[r];
		cuba_pose_round& c = rounds[r];
		c.iterations = s.iterations;
		c.kernel_type[0] = static_cast<int32_t>(s.kernelMono); c.kernel_type[1] = static_cast<int32_t>(s.kernelStereo);
		c.delta[0] = s.deltaMono; c.delta[1] = s.deltaStereo;
		c.restart = s.restart ? 1 : 0;
		c.chi2_mono = s.test.chi2Mono; c.chi2_stereo = s.test.chi2Stereo;
		c.flags = (s.test.requirePositiveDepth ? CUBA_CLASSIFY_DEPTH : 0) | (s.test.reinclude ? CUBA_CLASSIFY_REINCLUDE : 0);
		perProblem += static_cast<size_t>(std::max(s.iterations, 0));
	}
	return rounds;
}

// problem b's BatchStatistics per round
static std::vector<BatchStatistics> round_stats(const std::vector<cuba_pose_round>& rounds, const std::vector<cuba_iter_stat>& stats,
	const std::vector<int32_t>& nstats, size_t b, size_t perProblem)
{
	const size_t R = rounds.size();
	std::vector<BatchStatistics> out;
	size_t off = 0;
	for (size_t r = 0; r < R; r++) {
		BatchStatistics st;
		for (int i = 0; i < nstats[b * R + r]; i++) {
			const cuba_iter_stat& s = stats[b * perProblem + off + i];
			st.push_back(BatchInfo{ s.iteration, s.chi2 });
		}
		out.push_back(st);
		off += static_cast<size_t>(rounds[r].iterations);
	}
	return out;
}

std::vector<PoseResult> optimizePoses(CudaBundleAdjustment& ba, const std::vector<PoseFrame>& frames, const std::vector<PoseRound>& schedule)
{
	Impl& impl = impl_of(ba);
	if (frames.size() > static_cast<size_t>(INT32_MAX)) throw std::invalid_argument("cuba::optimizePoses: too many frames");
	const size_t B = frames.size();
	std::vector<double> q(4 * B), t(3 * B), cam(5 * B), X2, m2, om2, X3, m3, om3;
	std::vector<int32_t> ptr2(B + 1, 0), ptr3(B + 1, 0);
	for (size_t b = 0; b < B; b++) {
		const PoseFrame& f = frames[b];
		if (!f.pose) throw std::invalid_argument("cuba::optimizePoses: frame without a pose");
		for (int k = 0; k < 4; k++) q[4 * b + k] = f.pose->q.coeffs().data()[k];
		for (int k = 0; k < 3; k++) t[3 * b + k] = f.pose->t.data()[k];
		const CameraParams& c = f.pose->camera;
		cam[5 * b] = c.fx; cam[5 * b + 1] = c.fy; cam[5 * b + 2] = c.cx; cam[5 * b + 3] = c.cy; cam[5 * b + 4] = c.bf;
		for (const BaseEdge* e : f.edges) {
			if (!e) throw std::invalid_argument("cuba::optimizePoses: null edge");
			if (e->poseVertex() != f.pose) throw std::invalid_argument("cuba::optimizePoses: an edge's pose vertex is not the frame's pose");
			const LandmarkVertex* l = e->landmarkVertex();
			if (!l) throw std::invalid_argument("cuba::optimizePoses: an edge without a landmark");
			if (e->dim() == 2) {
				const MonoEdge* me = static_cast<const MonoEdge*>(e);
				for (int k = 0; k < 3; k++) X2.push_back(l->Xw.data()[k]);
				m2.push_back(me->measurement.data()[0]); m2.push_back(me->measurement.data()[1]);
				om2.push_back(me->information);
			} else if (e->dim() == 3) {
				const StereoEdge* se = static_cast<const StereoEdge*>(e);
				for (int k = 0; k < 3; k++) X3.push_back(l->Xw.data()[k]);
				for (int k = 0; k < 3; k++) m3.push_back(se->measurement.data()[k]);
				om3.push_back(se->information);
			} else throw std::invalid_argument("cuba::optimizePoses: an edge that is neither monocular nor stereo");
		}
		if (om2.size() + om3.size() > static_cast<size_t>(INT32_MAX)) throw std::invalid_argument("cuba::optimizePoses: too many edges");
		ptr2[b + 1] = static_cast<int32_t>(om2.size()); ptr3[b + 1] = static_cast<int32_t>(om3.size());
	}
	size_t perFrame = 0;
	const std::vector<cuba_pose_round> rounds = c_rounds(schedule, perFrame);
	const size_t R = rounds.size();
	cuba_pose_batch bt;
	bt.B = static_cast<int32_t>(B); bt.E2 = static_cast<int32_t>(om2.size()); bt.E3 = static_cast<int32_t>(om3.size());
	bt.q = q.data(); bt.t = t.data(); bt.cam = cam.data();
	bt.ptr2 = ptr2.data(); bt.X2 = X2.data(); bt.meas2 = m2.data(); bt.omega2 = om2.data();
	bt.ptr3 = ptr3.data(); bt.X3 = X3.data(); bt.meas3 = m3.data(); bt.omega3 = om3.data();
	std::vector<double> qo(4 * B), to(3 * B);
	std::vector<uint8_t> lev(om2.size() + om3.size());
	std::vector<int32_t> counts(4 * B * std::max<size_t>(R, 1)), nstats(B * std::max<size_t>(R, 1));
	std::vector<cuba_iter_stat> stats(std::max<size_t>(B * perFrame, 1));
	// the schedule and the batch are checked by the engine before anything runs: a refusal is the caller's input
	const int rc = cuba_engine_optimize_poses(impl.poseEngine(), &bt, static_cast<int>(R), rounds.data(), qo.data(), to.data(), lev.data(),
		counts.data(), stats.data(), nstats.data());
	if (rc == CUBA_ERR_INVALID) throw std::invalid_argument(std::string("cuba::optimizePoses: ") + cuba_last_error());
	if (rc != CUBA_OK) throw std::runtime_error(std::string("cuba_b200: ") + cuba_last_error());
	std::vector<PoseResult> out(B);
	const size_t E2 = om2.size();
	for (size_t b = 0; b < B; b++) {
		PoseVertex* p = frames[b].pose;
		for (int k = 0; k < 4; k++) p->q.coeffs().data()[k] = qo[4 * b + k];
		for (int k = 0; k < 3; k++) p->t.data()[k] = to[3 * b + k];
		PoseResult& res = out[b];
		size_t i2 = static_cast<size_t>(ptr2[b]), i3 = E2 + static_cast<size_t>(ptr3[b]);
		for (const BaseEdge* e : frames[b].edges) {
			const int lv = e->dim() == 2 ? lev[i2++] : lev[i3++];
			res.levels.push_back(lv);
			res.inliers += lv == 0;
		}
		res.rounds = round_stats(rounds, stats, nstats, b, perFrame);
	}
	return out;
}

// include/cuba_b200_points.h
std::vector<PointResult> optimizePoints(CudaBundleAdjustment& ba, const std::vector<PointProblem>& points, const std::vector<PoseRound>& schedule)
{
	Impl& impl = impl_of(ba);
	if (points.size() > static_cast<size_t>(INT32_MAX)) throw std::invalid_argument("cuba::optimizePoints: too many points");
	const size_t B = points.size();
	std::vector<double> Xw(3 * B), q, t, cam, m2, om2, m3, om3;
	std::vector<int32_t> ptr2(B + 1, 0), ptr3(B + 1, 0), iP2, iP3;
	std::unordered_map<const PoseVertex*, int32_t> table;    // each pose once, shared by every point that observes it
	for (size_t b = 0; b < B; b++) {
		const PointProblem& pt = points[b];
		if (!pt.landmark) throw std::invalid_argument("cuba::optimizePoints: point without a landmark");
		for (int k = 0; k < 3; k++) Xw[3 * b + k] = pt.landmark->Xw.data()[k];
		for (const BaseEdge* e : pt.edges) {
			if (!e) throw std::invalid_argument("cuba::optimizePoints: null edge");
			if (e->landmarkVertex() != pt.landmark) throw std::invalid_argument("cuba::optimizePoints: an edge's landmark vertex is not the point's landmark");
			const PoseVertex* p = e->poseVertex();
			if (!p) throw std::invalid_argument("cuba::optimizePoints: an edge without a pose");
			auto it = table.find(p);
			if (it == table.end()) {
				if (table.size() >= static_cast<size_t>(INT32_MAX)) throw std::invalid_argument("cuba::optimizePoints: too many poses");
				it = table.emplace(p, static_cast<int32_t>(table.size())).first;
				for (int k = 0; k < 4; k++) q.push_back(p->q.coeffs().data()[k]);
				for (int k = 0; k < 3; k++) t.push_back(p->t.data()[k]);
				const CameraParams& c = p->camera;
				cam.push_back(c.fx); cam.push_back(c.fy); cam.push_back(c.cx); cam.push_back(c.cy); cam.push_back(c.bf);
			}
			if (e->dim() == 2) {
				const MonoEdge* me = static_cast<const MonoEdge*>(e);
				m2.push_back(me->measurement.data()[0]); m2.push_back(me->measurement.data()[1]);
				om2.push_back(me->information);
				iP2.push_back(it->second);
			} else if (e->dim() == 3) {
				const StereoEdge* se = static_cast<const StereoEdge*>(e);
				for (int k = 0; k < 3; k++) m3.push_back(se->measurement.data()[k]);
				om3.push_back(se->information);
				iP3.push_back(it->second);
			} else throw std::invalid_argument("cuba::optimizePoints: an edge that is neither monocular nor stereo");
		}
		if (om2.size() + om3.size() > static_cast<size_t>(INT32_MAX)) throw std::invalid_argument("cuba::optimizePoints: too many edges");
		ptr2[b + 1] = static_cast<int32_t>(om2.size()); ptr3[b + 1] = static_cast<int32_t>(om3.size());
	}
	size_t perPoint = 0;
	const std::vector<cuba_pose_round> rounds = c_rounds(schedule, perPoint);
	const size_t R = rounds.size();
	cuba_point_batch bt;
	bt.B = static_cast<int32_t>(B); bt.P = static_cast<int32_t>(table.size());
	bt.E2 = static_cast<int32_t>(om2.size()); bt.E3 = static_cast<int32_t>(om3.size());
	bt.Xw = Xw.data(); bt.q = q.data(); bt.t = t.data(); bt.cam = cam.data();
	bt.ptr2 = ptr2.data(); bt.iP2 = iP2.data(); bt.meas2 = m2.data(); bt.omega2 = om2.data();
	bt.ptr3 = ptr3.data(); bt.iP3 = iP3.data(); bt.meas3 = m3.data(); bt.omega3 = om3.data();
	std::vector<double> Xo(3 * B);
	std::vector<uint8_t> lev(om2.size() + om3.size());
	std::vector<int32_t> counts(4 * B * std::max<size_t>(R, 1)), nstats(B * std::max<size_t>(R, 1));
	std::vector<cuba_iter_stat> stats(std::max<size_t>(B * perPoint, 1));
	// the schedule and the batch are checked by the engine before anything runs: a refusal is the caller's input
	const int rc = cuba_engine_optimize_points(impl.poseEngine(), &bt, static_cast<int>(R), rounds.data(), Xo.data(), lev.data(), counts.data(),
		stats.data(), nstats.data());
	if (rc == CUBA_ERR_INVALID) throw std::invalid_argument(std::string("cuba::optimizePoints: ") + cuba_last_error());
	if (rc != CUBA_OK) throw std::runtime_error(std::string("cuba_b200: ") + cuba_last_error());
	std::vector<PointResult> out(B);
	const size_t E2 = om2.size();
	for (size_t b = 0; b < B; b++) {
		LandmarkVertex* l = points[b].landmark;
		for (int k = 0; k < 3; k++) l->Xw.data()[k] = Xo[3 * b + k];
		PointResult& res = out[b];
		size_t i2 = static_cast<size_t>(ptr2[b]), i3 = E2 + static_cast<size_t>(ptr3[b]);
		for (const BaseEdge* e : points[b].edges) {
			const int lv = e->dim() == 2 ? lev[i2++] : lev[i3++];
			res.levels.push_back(lv);
			res.inliers += lv == 0;
		}
		res.rounds = round_stats(rounds, stats, nstats, b, perPoint);
	}
	return out;
}

std::vector<OutlierCounts> optimizeLandmarks(CudaBundleAdjustment& ba, const std::vector<PoseRound>& schedule)
{
	size_t per = 0;
	return impl_of(ba).optimizeLandmarks(c_rounds(schedule, per), nullptr);
}
std::vector<OutlierCounts> optimizeLandmarks(CudaBundleAdjustment& ba, const std::vector<PoseRound>& schedule,
	const std::vector<LandmarkVertex*>& landmarks)
{
	size_t per = 0;
	return impl_of(ba).optimizeLandmarks(c_rounds(schedule, per), &landmarks);
}

// include/cuba_b200_sim3.h
std::vector<Sim3Result> optimizeSim3(CudaBundleAdjustment& ba, const std::vector<Sim3Problem>& problems, const Sim3Options& options)
{
	Impl& impl = impl_of(ba);
	if (problems.size() > static_cast<size_t>(INT32_MAX)) throw std::invalid_argument("cuba::optimizeSim3: too many problems");
	const size_t B = problems.size();
	std::vector<double> q(4 * B), t(3 * B), s(B), cam1(4 * B), cam2(4 * B), X1, X2, o1, o2, om1, om2;
	std::vector<int32_t> ptr(B + 1, 0), fix(B);
	for (size_t b = 0; b < B; b++) {
		const Sim3Problem& p = problems[b];
		for (int k = 0; k < 4; k++) q[4 * b + k] = p.q.coeffs().data()[k];
		for (int k = 0; k < 3; k++) t[3 * b + k] = p.t.data()[k];
		s[b] = p.s;
		const CameraParams* c[2] = { &p.camera1, &p.camera2 };
		double* cd[2] = { cam1.data() + 4 * b, cam2.data() + 4 * b };
		for (int k = 0; k < 2; k++) { cd[k][0] = c[k]->fx; cd[k][1] = c[k]->fy; cd[k][2] = c[k]->cx; cd[k][3] = c[k]->cy; }
		fix[b] = p.fixScale ? 1 : 0;
		for (const Sim3Match& m : p.matches) {
			for (int k = 0; k < 3; k++) { X1.push_back(m.X1.data()[k]); X2.push_back(m.X2.data()[k]); }
			for (int k = 0; k < 2; k++) { o1.push_back(m.obs1.data()[k]); o2.push_back(m.obs2.data()[k]); }
			om1.push_back(m.information1); om2.push_back(m.information2);
		}
		if (om1.size() > static_cast<size_t>(INT32_MAX)) throw std::invalid_argument("cuba::optimizeSim3: too many matches");
		ptr[b + 1] = static_cast<int32_t>(om1.size());
	}
	const size_t N = om1.size();
	cuba_sim3_batch bt;
	bt.B = static_cast<int32_t>(B); bt.N = static_cast<int32_t>(N); bt.ptr = ptr.data();
	bt.q = q.data(); bt.t = t.data(); bt.s = s.data(); bt.cam1 = cam1.data(); bt.cam2 = cam2.data(); bt.fix_scale = fix.data();
	bt.X1 = X1.data(); bt.X2 = X2.data(); bt.obs1 = o1.data(); bt.obs2 = o2.data(); bt.omega1 = om1.data(); bt.omega2 = om2.data();
	cuba_sim3_params prm;
	prm.chi2 = options.chi2; prm.iterations = options.iterations; prm.iterations_bad = options.iterationsBad;
	prm.iterations_good = options.iterationsGood; prm.min_pairs = options.minPairs;
	const size_t perProblem = static_cast<size_t>(std::max(options.iterations, 0)) +
		static_cast<size_t>(std::max(std::max(options.iterationsBad, options.iterationsGood), 0));
	std::vector<double> qo(4 * B), to(3 * B), so(B);
	std::vector<uint8_t> lev(N);
	std::vector<int32_t> inl(B), nstats(2 * B);
	std::vector<cuba_iter_stat> stats(std::max<size_t>(B * perProblem, 1));
	// the options and the batch are checked by the engine before anything runs: a refusal is the caller's input
	const int rc = cuba_engine_optimize_sim3(impl.poseEngine(), &bt, &prm, qo.data(), to.data(), so.data(), lev.data(), inl.data(),
		stats.data(), nstats.data());
	if (rc == CUBA_ERR_INVALID) throw std::invalid_argument(std::string("cuba::optimizeSim3: ") + cuba_last_error());
	if (rc != CUBA_OK) throw std::runtime_error(std::string("cuba_b200: ") + cuba_last_error());
	std::vector<Sim3Result> out(B);
	for (size_t b = 0; b < B; b++) {
		Sim3Result& r = out[b];
		for (int k = 0; k < 4; k++) r.q.coeffs().data()[k] = qo[4 * b + k];
		for (int k = 0; k < 3; k++) r.t.data()[k] = to[3 * b + k];
		r.s = so[b];
		r.inliers = static_cast<size_t>(inl[b]);
		for (size_t i = static_cast<size_t>(ptr[b]); i < static_cast<size_t>(ptr[b + 1]); i++) r.levels.push_back(lev[i]);
		for (int k = 0; k < 2; k++) {
			BatchStatistics st;
			const size_t off = b * perProblem + (k ? static_cast<size_t>(options.iterations) : 0);
			for (int i = 0; i < nstats[2 * b + k]; i++) st.push_back(BatchInfo{ stats[off + i].iteration, stats[off + i].chi2 });
			r.rounds.push_back(st);
		}
	}
	return out;
}

static bool dropin_levels(CudaBundleAdjustment* obj, const uint8_t** levels, int32_t* n)
{
	Impl* impl = dynamic_cast<Impl*>(obj);
	return impl && impl->flatLevels(levels, n);
}

} // namespace cuba

extern "C" int cuba_debug_dropin_problem(void* dropin, cuba_problem* out)
{
	return cuba::dropin_problem(static_cast<cuba::CudaBundleAdjustment*>(dropin), out) ? CUBA_OK : CUBA_ERR_STATE;
}

extern "C" int cuba_debug_dropin_levels(void* dropin, const uint8_t** levels, int32_t* n)
{
	try {
		return cuba::dropin_levels(static_cast<cuba::CudaBundleAdjustment*>(dropin), levels, n) ? CUBA_OK : CUBA_ERR_STATE;
	} catch (const std::exception&) {
		return CUBA_ERR_CUDA;      // fetching classifyEdges() decisions failed (cuba_last_error has the message)
	}
}
