// pose_batch_driver.cpp -- TEST DRIVER for cuba::optimizePoses (include/cuba_b200_pose.h).
//   pose_batch_driver frames.cubagraph other.cubagraph
// Every pose of frames.cubagraph becomes one frame with all of its edges (stereo edges first, then mono, to exercise the mapping of
// levels back to the frame's edge order), optimised under orbSlam2PoseSchedule().  The optimizer object holds other.cubagraph, an
// unrelated graph: its initialize() + optimize(10) runs before and after the batch from the same estimate and must not change.
// Prints one JSON object; tests/test_pose_batch.py checks it against the CPU oracle.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include <cuba_b200.h>
#include <cuba_b200_pose.h>

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
	if (argc < 3) { fprintf(stderr, "usage: pose_batch_driver frames.cubagraph other.cubagraph\n"); return 2; }
	Storage fs;
	auto holder = readGraph(argv[1], fs);      // owns nothing the batch needs: frames are built from the vertices and edges directly
	Storage os;
	auto ba = readGraph(argv[2], os);
	Snapshot start, end1, end2;
	start.take(os);
	const std::vector<double> chiBefore = runOther(*ba, os, start, end1);

	std::vector<cuba::PoseFrame> frames(fs.poses.size());
	for (size_t p = 0; p < fs.poses.size(); p++) {
		frames[p].pose = fs.poses[p].get();
		for (auto& e : fs.stereo) if (e->vertexP == frames[p].pose) frames[p].edges.push_back(e.get());
		for (auto& e : fs.mono) if (e->vertexP == frames[p].pose) frames[p].edges.push_back(e.get());
	}
	const std::vector<cuba::PoseResult> res = cuba::optimizePoses(*ba, frames);

	const std::vector<double> chiAfter = runOther(*ba, os, start, end2);

	// malformed input: an edge of another pose, and an out-of-range schedule
	bool threwPose = false, threwSchedule = false;
	if (frames.size() >= 2 && !frames[1].edges.empty()) {
		std::vector<cuba::PoseFrame> bad(1, frames[0]);
		bad[0].edges.push_back(frames[1].edges[0]);
		try { cuba::optimizePoses(*ba, bad); } catch (const std::invalid_argument&) { threwPose = true; }
	}
	try { cuba::optimizePoses(*ba, frames, std::vector<cuba::PoseRound>(9)); } catch (const std::invalid_argument&) { threwSchedule = true; }

	printf("{\"frames\": [");
	for (size_t b = 0; b < res.size(); b++) {
		const cuba::PoseVertex* p = frames[b].pose;
		printf("%s{\"id\": %d, \"q\": [%.17g, %.17g, %.17g, %.17g], \"t\": [%.17g, %.17g, %.17g], \"inliers\": %zu, \"edges\": [", b ? ", " : "", p->id,
			p->q.coeffs().data()[0], p->q.coeffs().data()[1], p->q.coeffs().data()[2], p->q.coeffs().data()[3], p->t.data()[0], p->t.data()[1], p->t.data()[2],
			res[b].inliers);
		// each edge as [stereo, file row, level]
		for (size_t k = 0; k < frames[b].edges.size(); k++) {
			const cuba::BaseEdge* e = frames[b].edges[k];
			long row = -1;
			if (e->dim() == 3) { for (size_t i = 0; i < fs.stereo.size(); i++) if (fs.stereo[i].get() == e) row = (long)i; }
			else { for (size_t i = 0; i < fs.mono.size(); i++) if (fs.mono[i].get() == e) row = (long)i; }
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
	printf("], \"other_state_equal\": %s, \"threw_pose\": %s, \"threw_schedule\": %s}\n", end1.v == end2.v ? "true" : "false",
		threwPose ? "true" : "false", threwSchedule ? "true" : "false");
	(void)holder;
	return 0;
}
