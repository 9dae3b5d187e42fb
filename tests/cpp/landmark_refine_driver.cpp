// landmark_refine_driver.cpp -- TEST DRIVER for cuba::optimizeLandmarks (include/cuba_b200_points.h).
//   landmark_refine_driver graph.cubagraph
// The graph is optimised (optimize(5)); then every other free landmark is refined in place with a list, and afterwards every free
// landmark without one, every edge back at level 0 first.  Before each call cuba::optimizePoints runs on the same landmarks from the
// same positions (every edge at level 0, the vertices' poses as they stand), and the vertices are put back: its Xw and levels are
// the reference of the in-place call's.  Two refusals: a call before any optimize(), and a fixed landmark in the list.
// Prints one JSON object; tests/test_landmark_refine.py compares the two.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include <cuba_b200.h>
#include <cuba_b200_points.h>

#include "../../samples/cubagraph_reader.h"

static std::vector<cuba::PoseRound> schedule()
{
	std::vector<cuba::PoseRound> s(2);
	s[0].iterations = 5;
	s[0].kernelMono = s[0].kernelStereo = cuba::RobustKernelType::HUBER;
	s[0].deltaMono = std::sqrt(5.991); s[0].deltaStereo = std::sqrt(7.815);
	s[0].restart = false;
	s[0].test.requirePositiveDepth = true; s[0].test.reinclude = false;
	s[1].iterations = 10;
	s[1].restart = false;
	s[1].test.requirePositiveDepth = true; s[1].test.reinclude = true;
	return s;
}

// one run: the in-place call on `list` (all free landmarks when `all`), against cuba::optimizePoints from the same start
static void run(cuba::CudaBundleAdjustment& ba, Storage& st, const std::vector<cuba::LandmarkVertex*>& list, bool all, bool comma)
{
	std::vector<cuba::PointProblem> pts(list.size());
	std::vector<double> start;
	for (size_t b = 0; b < list.size(); b++) {
		pts[b].landmark = list[b];
		for (auto& e : st.mono) if (e->vertexL == list[b]) pts[b].edges.push_back(e.get());
		for (auto& e : st.stereo) if (e->vertexL == list[b]) pts[b].edges.push_back(e.get());
		for (int k = 0; k < 3; k++) start.push_back(list[b]->Xw.data()[k]);
	}
	const std::vector<cuba::PointResult> ref = cuba::optimizePoints(ba, pts, schedule());
	std::vector<double> refX;
	for (size_t b = 0; b < list.size(); b++)
		for (int k = 0; k < 3; k++) { refX.push_back(list[b]->Xw.data()[k]); list[b]->Xw.data()[k] = start[3 * b + k]; }
	const std::vector<cuba::OutlierCounts> c = all ? cuba::optimizeLandmarks(ba, schedule()) : cuba::optimizeLandmarks(ba, schedule(), list);
	printf("%s{\"all\": %s, \"counts\": [", comma ? ", " : "", all ? "true" : "false");
	for (size_t r = 0; r < c.size(); r++)
		printf("%s[%zu, %zu, %zu, %zu]", r ? ", " : "", c[r].includedMono, c[r].includedStereo, c[r].excluded, c[r].reincluded);
	printf("], \"points\": [");
	for (size_t b = 0; b < list.size(); b++) {
		const double* x = list[b]->Xw.data();
		printf("%s{\"id\": %d, \"Xw\": [%.17g, %.17g, %.17g], \"ref\": [%.17g, %.17g, %.17g], \"levels\": [", b ? ", " : "", list[b]->id,
			x[0], x[1], x[2], refX[3 * b], refX[3 * b + 1], refX[3 * b + 2]);
		for (size_t k = 0; k < pts[b].edges.size(); k++)
			printf("%s[%d, %d]", k ? ", " : "", cuba::edgeLevel(ba, pts[b].edges[k]), ref[b].levels[k]);
		printf("]}");
	}
	printf("]}");
}

int main(int argc, char** argv)
{
	if (argc < 2) { fprintf(stderr, "usage: landmark_refine_driver graph.cubagraph\n"); return 2; }
	Storage st;
	auto ba = readGraph(argv[1], st);
	ba->setRobustKernels(cuba::RobustKernelType::HUBER, std::sqrt(5.991), cuba::EdgeType::MONOCULAR);
	ba->setRobustKernels(cuba::RobustKernelType::HUBER, std::sqrt(7.815), cuba::EdgeType::STEREO);
	ba->initialize();
	bool threwState = false, threwFixed = false;
	try { cuba::optimizeLandmarks(*ba, schedule()); } catch (const std::logic_error&) { threwState = true; }
	ba->optimize(5);

	std::vector<cuba::LandmarkVertex*> half, every;
	cuba::LandmarkVertex* fixedOne = nullptr;
	for (auto& l : st.landmarks) {
		if (l->fixed) { if (!fixedOne) fixedOne = l.get(); continue; }
		if (l->edges.empty()) continue;
		if (every.size() % 2 == 0) half.push_back(l.get());
		every.push_back(l.get());
	}
	printf("{\"runs\": [");
	run(*ba, st, half, false, false);
	for (auto& e : st.mono) cuba::setEdgeLevel(*ba, e.get(), 0);
	for (auto& e : st.stereo) cuba::setEdgeLevel(*ba, e.get(), 0);
	run(*ba, st, every, true, true);
	if (fixedOne) {
		try { cuba::optimizeLandmarks(*ba, schedule(), std::vector<cuba::LandmarkVertex*>(1, fixedOne)); }
		catch (const std::invalid_argument&) { threwFixed = true; }
	}
	printf("], \"threw_state\": %s, \"threw_fixed\": %s, \"has_fixed\": %s}\n", threwState ? "true" : "false", threwFixed ? "true" : "false",
		fixedOne ? "true" : "false");
	return 0;
}
