// sim3_batch_driver.cpp -- TEST DRIVER for cuba::optimizeSim3 (include/cuba_b200_sim3.h).
//   sim3_batch_driver problems.txt other.cubagraph
// problems.txt: the number of problems, then per problem "q(4) t(3) s cam1(4) cam2(4) fixScale N" and N lines "X1(3) X2(3) obs1(2)
// obs2(2) information1 information2".  They run under the default options on an optimizer that holds other.cubagraph, an unrelated
// graph: its initialize() + optimize(10) runs before and after the batch from the same estimate and must not change.  Prints one JSON
// object; tests/test_sim3_batch.py compares it with Engine.optimize_sim3.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include <cuba_b200.h>
#include <cuba_b200_sim3.h>

#include "../../samples/cubagraph_reader.h"

static std::vector<double> runOther(cuba::CudaBundleAdjustment& ba, Storage& st, const std::vector<double>& start, std::vector<double>& end)
{
	size_t i = 0;
	for (auto& p : st.poses) { for (int k = 0; k < 4; k++) p->q.coeffs().data()[k] = start[i++]; for (int k = 0; k < 3; k++) p->t.data()[k] = start[i++]; }
	for (auto& l : st.landmarks) for (int k = 0; k < 3; k++) l->Xw.data()[k] = start[i++];
	ba.initialize();
	const size_t before = ba.batchStatistics().size();
	ba.optimize(10);
	std::vector<double> chi;
	for (size_t k = before; k < ba.batchStatistics().size(); k++) chi.push_back(ba.batchStatistics()[k].chi2);
	end.clear();
	for (auto& p : st.poses) { for (int k = 0; k < 4; k++) end.push_back(p->q.coeffs().data()[k]); for (int k = 0; k < 3; k++) end.push_back(p->t.data()[k]); }
	for (auto& l : st.landmarks) for (int k = 0; k < 3; k++) end.push_back(l->Xw.data()[k]);
	return chi;
}

static double rdv(FILE* f)
{
	double v;
	if (fscanf(f, "%lf", &v) != 1) throw std::runtime_error("short problems file");
	return v;
}

int main(int argc, char** argv)
{
	if (argc < 3) { fprintf(stderr, "usage: sim3_batch_driver problems.txt other.cubagraph\n"); return 2; }
	FILE* f = fopen(argv[1], "r");
	if (!f) { fprintf(stderr, "cannot open %s\n", argv[1]); return 2; }
	std::vector<cuba::Sim3Problem> problems(static_cast<size_t>(rdv(f)));
	for (cuba::Sim3Problem& p : problems) {
		for (int k = 0; k < 4; k++) p.q.coeffs().data()[k] = rdv(f);
		for (int k = 0; k < 3; k++) p.t.data()[k] = rdv(f);
		p.s = rdv(f);
		p.camera1.fx = rdv(f); p.camera1.fy = rdv(f); p.camera1.cx = rdv(f); p.camera1.cy = rdv(f);
		p.camera2.fx = rdv(f); p.camera2.fy = rdv(f); p.camera2.cx = rdv(f); p.camera2.cy = rdv(f);
		p.fixScale = rdv(f) != 0;
		p.matches.resize(static_cast<size_t>(rdv(f)));
		for (cuba::Sim3Match& m : p.matches) {
			for (int k = 0; k < 3; k++) m.X1.data()[k] = rdv(f);
			for (int k = 0; k < 3; k++) m.X2.data()[k] = rdv(f);
			for (int k = 0; k < 2; k++) m.obs1.data()[k] = rdv(f);
			for (int k = 0; k < 2; k++) m.obs2.data()[k] = rdv(f);
			m.information1 = rdv(f); m.information2 = rdv(f);
		}
	}
	fclose(f);

	Storage os;
	auto ba = readGraph(argv[2], os);
	std::vector<double> start, end1, end2;
	for (auto& p : os.poses) { for (int k = 0; k < 4; k++) start.push_back(p->q.coeffs().data()[k]); for (int k = 0; k < 3; k++) start.push_back(p->t.data()[k]); }
	for (auto& l : os.landmarks) for (int k = 0; k < 3; k++) start.push_back(l->Xw.data()[k]);
	const std::vector<double> chiBefore = runOther(*ba, os, start, end1);
	const std::vector<cuba::Sim3Result> res = cuba::optimizeSim3(*ba, problems);
	const std::vector<double> chiAfter = runOther(*ba, os, start, end2);

	// malformed input: s <= 0, and options the engine refuses
	bool threwScale = false, threwOptions = false;
	if (!problems.empty()) {
		std::vector<cuba::Sim3Problem> bad(1, problems[0]);
		bad[0].s = 0;
		try { cuba::optimizeSim3(*ba, bad); } catch (const std::invalid_argument&) { threwScale = true; }
	}
	cuba::Sim3Options badOptions;
	badOptions.chi2 = -1;
	try { cuba::optimizeSim3(*ba, problems, badOptions); } catch (const std::invalid_argument&) { threwOptions = true; }

	printf("{\"problems\": [");
	for (size_t b = 0; b < res.size(); b++) {
		const cuba::Sim3Result& r = res[b];
		printf("%s{\"q\": [%.17g, %.17g, %.17g, %.17g], \"t\": [%.17g, %.17g, %.17g], \"s\": %.17g, \"inliers\": %zu, \"levels\": [", b ? ", " : "",
			r.q.coeffs().data()[0], r.q.coeffs().data()[1], r.q.coeffs().data()[2], r.q.coeffs().data()[3], r.t.data()[0], r.t.data()[1], r.t.data()[2],
			r.s, r.inliers);
		for (size_t k = 0; k < r.levels.size(); k++) printf("%s%d", k ? ", " : "", r.levels[k]);
		printf("], \"rounds\": [");
		for (size_t k = 0; k < r.rounds.size(); k++) {
			printf("%s[", k ? ", " : "");
			for (size_t i = 0; i < r.rounds[k].size(); i++) printf("%s%.17g", i ? ", " : "", r.rounds[k][i].chi2);
			printf("]");
		}
		printf("]}");
	}
	printf("], \"other_before\": [");
	for (size_t i = 0; i < chiBefore.size(); i++) printf("%s%.17g", i ? ", " : "", chiBefore[i]);
	printf("], \"other_after\": [");
	for (size_t i = 0; i < chiAfter.size(); i++) printf("%s%.17g", i ? ", " : "", chiAfter[i]);
	printf("], \"other_state_equal\": %s, \"threw_scale\": %s, \"threw_options\": %s}\n", end1 == end2 ? "true" : "false",
		threwScale ? "true" : "false", threwOptions ? "true" : "false");
	return 0;
}
