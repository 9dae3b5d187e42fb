// point_batch_driver.cpp -- TEST DRIVER for cuba::optimizePoints (include/cuba_b200_points.h).
//   point_batch_driver points.cubagraph other.cubagraph
// Every landmark of points.cubagraph becomes one point with all of its edges (stereo edges first, then mono, to exercise the mapping
// of levels back to the point's edge order), refined under two rounds: Huber 5 iterations with the depth test, then no robust kernel
// 10 iterations with the depth test and re-inclusion, each from the last round's result.  The optimizer object holds other.cubagraph,
// an unrelated graph: its initialize() + optimize(10) runs before and after the batch from the same estimate and must not change.
// Prints one JSON object; tests/test_point_batch.py checks it against Engine.optimize_points.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include <cuba_b200.h>
#include <cuba_b200_points.h>

#include "../../samples/cubagraph_reader.h"

struct Snapshot {
	std::vector<double> v;
	void take(const Storage& st)
	{
		v.clear();
		for (auto& p : st.poses) { for (int k = 0; k < 4; k++) v.push_back(p->q.coeffs().data()[k]); for (int k = 0; k < 3; k++) v.push_back(p->t.data()[k]); }
		for (auto& l : st.landmarks) for (int k = 0; k < 3; k++) v.push_back(l->Xw.data()[k]);
	}
	void restore(Storage& st) const
	{
		size_t i = 0;
		for (auto& p : st.poses) { for (int k = 0; k < 4; k++) p->q.coeffs().data()[k] = v[i++]; for (int k = 0; k < 3; k++) p->t.data()[k] = v[i++]; }
		for (auto& l : st.landmarks) for (int k = 0; k < 3; k++) l->Xw.data()[k] = v[i++];
	}
};

static std::vector<double> runOther(cuba::CudaBundleAdjustment& ba, Storage& st, const Snapshot& start, Snapshot& end)
{
	start.restore(st);
	ba.setRobustKernels(cuba::RobustKernelType::HUBER, std::sqrt(5.991), cuba::EdgeType::MONOCULAR);
	ba.setRobustKernels(cuba::RobustKernelType::HUBER, std::sqrt(7.815), cuba::EdgeType::STEREO);
	ba.initialize();
	const size_t before = ba.batchStatistics().size();
	ba.optimize(10);
	std::vector<double> chi;
	for (size_t i = before; i < ba.batchStatistics().size(); i++) chi.push_back(ba.batchStatistics()[i].chi2);
	end.take(st);
	return chi;
}

int main(int argc, char** argv)
{
	if (argc < 3) { fprintf(stderr, "usage: point_batch_driver points.cubagraph other.cubagraph\n"); return 2; }
	Storage ps;
	auto holder = readGraph(argv[1], ps);      // owns nothing the batch needs: points are built from the vertices and edges directly
	Storage os;
	auto ba = readGraph(argv[2], os);
	Snapshot start, end1, end2;
	start.take(os);
	const std::vector<double> chiBefore = runOther(*ba, os, start, end1);

	std::vector<cuba::PointProblem> points(ps.landmarks.size());
	for (size_t l = 0; l < ps.landmarks.size(); l++) {
		points[l].landmark = ps.landmarks[l].get();
		for (auto& e : ps.stereo) if (e->vertexL == points[l].landmark) points[l].edges.push_back(e.get());
		for (auto& e : ps.mono) if (e->vertexL == points[l].landmark) points[l].edges.push_back(e.get());
	}
	std::vector<cuba::PoseRound> schedule(2);
	schedule[0].iterations = 5;
	schedule[0].kernelMono = schedule[0].kernelStereo = cuba::RobustKernelType::HUBER;
	schedule[0].deltaMono = std::sqrt(5.991); schedule[0].deltaStereo = std::sqrt(7.815);
	schedule[0].restart = false;
	schedule[0].test.requirePositiveDepth = true; schedule[0].test.reinclude = false;
	schedule[1].iterations = 10;
	schedule[1].restart = false;
	schedule[1].test.requirePositiveDepth = true; schedule[1].test.reinclude = true;
	const std::vector<cuba::PointResult> res = cuba::optimizePoints(*ba, points, schedule);

	const std::vector<double> chiAfter = runOther(*ba, os, start, end2);

	// malformed input: an edge of another landmark, and an out-of-range schedule
	bool threwLandmark = false, threwSchedule = false;
	if (points.size() >= 2 && !points[1].edges.empty()) {
		std::vector<cuba::PointProblem> bad(1, points[0]);
		bad[0].edges.push_back(points[1].edges[0]);
		try { cuba::optimizePoints(*ba, bad, schedule); } catch (const std::invalid_argument&) { threwLandmark = true; }
	}
	try { cuba::optimizePoints(*ba, points, std::vector<cuba::PoseRound>(9)); } catch (const std::invalid_argument&) { threwSchedule = true; }

	printf("{\"points\": [");
	for (size_t b = 0; b < res.size(); b++) {
		const cuba::LandmarkVertex* l = points[b].landmark;
		printf("%s{\"id\": %d, \"Xw\": [%.17g, %.17g, %.17g], \"inliers\": %zu, \"edges\": [", b ? ", " : "", l->id, l->Xw.data()[0], l->Xw.data()[1],
			l->Xw.data()[2], res[b].inliers);
		// each edge as [stereo, file row, level]
		for (size_t k = 0; k < points[b].edges.size(); k++) {
			const cuba::BaseEdge* e = points[b].edges[k];
			long row = -1;
			if (e->dim() == 3) { for (size_t i = 0; i < ps.stereo.size(); i++) if (ps.stereo[i].get() == e) row = (long)i; }
			else { for (size_t i = 0; i < ps.mono.size(); i++) if (ps.mono[i].get() == e) row = (long)i; }
			printf("%s[%d, %ld, %d]", k ? ", " : "", e->dim() == 3 ? 1 : 0, row, res[b].levels[k]);
		}
		printf("], \"rounds\": [");
		for (size_t r = 0; r < res[b].rounds.size(); r++) {
			printf("%s[", r ? ", " : "");
			for (size_t i = 0; i < res[b].rounds[r].size(); i++) printf("%s%.17g", i ? ", " : "", res[b].rounds[r][i].chi2);
			printf("]");
		}
		printf("]}");
	}
	printf("], \"other_before\": [");
	for (size_t i = 0; i < chiBefore.size(); i++) printf("%s%.17g", i ? ", " : "", chiBefore[i]);
	printf("], \"other_after\": [");
	for (size_t i = 0; i < chiAfter.size(); i++) printf("%s%.17g", i ? ", " : "", chiAfter[i]);
	printf("], \"other_state_equal\": %s, \"threw_landmark\": %s, \"threw_schedule\": %s}\n", end1.v == end2.v ? "true" : "false",
		threwLandmark ? "true" : "false", threwSchedule ? "true" : "false");
	(void)holder;
	return 0;
}
