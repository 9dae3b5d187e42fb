// levels_driver.cpp -- TEST DRIVER for the edge levels of the drop-in class (include/cuba_b200_levels.h).  Executes a ';'-separated
// op list on a .cubagraph and prints one JSON object; tests/test_edge_levels.py mirrors the ops on the graph arrays (bookkeeping
// without a GPU, ORB-SLAM2's outlier rounds against the CPU oracle).
//   init | opt:N | kernel:none|huber | level:m|s:K:L | rmedge:m|s:K | addedge:m|s:K | fixp:ID | unfixp:ID | fixl:ID | unfixl:ID
//   flat (the flat levels of cuba_debug_dropin_levels) | classify:CHI2MONO:CHI2STEREO:DEPTH:REINCLUDE | levels (edgeLevel of every edge)
#include <cmath>
#include <sstream>
#include <stdexcept>

#include <cuba_b200.h>
#include <cuba_b200_levels.h>

#include "../../samples/cubagraph_reader.h"

static void printLevels(const cuba::CudaBundleAdjustment& opt, const Storage& st)
{
	// per graph edge, file order: 0 / 1, or -1 for an edge the optimizer does not hold (std::out_of_range)
	auto one = [&](const cuba::BaseEdge* e) { try { return cuba::edgeLevel(opt, e); } catch (const std::out_of_range&) { return -1; } };
	printf(", \"mono_levels\": [");
	for (size_t i = 0; i < st.mono.size(); i++) printf("%s%d", i ? ", " : "", one(st.mono[i].get()));
	printf("], \"stereo_levels\": [");
	for (size_t i = 0; i < st.stereo.size(); i++) printf("%s%d", i ? ", " : "", one(st.stereo[i].get()));
	printf("]");
}

int main(int argc, char** argv)
{
	if (argc < 4) { fprintf(stderr, "usage: levels_driver graph.cubagraph ops dump.bin\n"); return 2; }
	Storage st;
	auto opt = readGraph(argv[1], st);
	std::stringstream ss(argv[2]);
	std::string op;
	printf("{\"steps\": [");
	bool first = true;
	while (std::getline(ss, op, ';')) {
		if (op.empty()) continue;
		std::vector<std::string> f;
		{ std::stringstream s2(op); std::string x; while (std::getline(s2, x, ':')) f.push_back(x); }
		printf("%s{\"op\": \"%s\"", first ? "" : ", ", op.c_str());
		first = false;
		auto edge = [&](const std::string& kind, const std::string& k) -> cuba::BaseEdge* {
			const size_t i = atol(k.c_str());
			return kind == "m" ? static_cast<cuba::BaseEdge*>(st.mono[i].get()) : static_cast<cuba::BaseEdge*>(st.stereo[i].get());
		};
		if (f[0] == "init") opt->initialize();
		else if (f[0] == "opt") {
			const size_t before = opt->batchStatistics().size();
			opt->optimize(atoi(f[1].c_str()));
			const auto& s = opt->batchStatistics();
			printf(", \"chi2\": [");
			for (size_t i = before; i < s.size(); i++) printf("%s%.17g", i > before ? ", " : "", s[i].chi2);
			printf("], \"mono_chi2\": [");
			for (size_t i = 0; i < st.mono.size(); i++) printf("%s%.17g", i ? ", " : "", opt->chiSquared(st.mono[i].get()));
			printf("], \"stereo_chi2\": [");
			for (size_t i = 0; i < st.stereo.size(); i++) printf("%s%.17g", i ? ", " : "", opt->chiSquared(st.stereo[i].get()));
			printf("]");
		}
		else if (f[0] == "kernel") {
			const bool huber = f[1] == "huber";
			opt->setRobustKernels(huber ? cuba::RobustKernelType::HUBER : cuba::RobustKernelType::NONE, huber ? std::sqrt(5.991) : 0.0, cuba::EdgeType::MONOCULAR);
			opt->setRobustKernels(huber ? cuba::RobustKernelType::HUBER : cuba::RobustKernelType::NONE, huber ? std::sqrt(7.815) : 0.0, cuba::EdgeType::STEREO);
		}
		else if (f[0] == "level") {
			bool threw = false;
			try { cuba::setEdgeLevel(*opt, edge(f[1], f[2]), atoi(f[3].c_str())); } catch (const std::out_of_range&) { threw = true; }
			printf(", \"threw\": %s", threw ? "true" : "false");
		}
		else if (f[0] == "rmedge") opt->removeEdge(edge(f[1], f[2]));
		else if (f[0] == "addedge") { if (f[1] == "m") opt->addMonocularEdge(st.mono[atol(f[2].c_str())].get()); else opt->addStereoEdge(st.stereo[atol(f[2].c_str())].get()); }
		else if (f[0] == "fixp" || f[0] == "unfixp") opt->poseVertex(atoi(f[1].c_str()))->fixed = f[0] == "fixp";
		else if (f[0] == "fixl" || f[0] == "unfixl") opt->landmarkVertex(atoi(f[1].c_str()))->fixed = f[0] == "fixl";
		else if (f[0] == "flat") {
			const uint8_t* lv = nullptr;
			int32_t n = 0;
			if (cuba_debug_dropin_levels(opt.get(), &lv, &n) != CUBA_OK) { fprintf(stderr, "cuba_debug_dropin_levels failed\n"); return 3; }
			printf(", \"flat\": [");
			for (int32_t i = 0; i < n; i++) printf("%s%d", i ? ", " : "", lv[i]);
			printf("]");
		}
		else if (f[0] == "classify") {
			cuba::OutlierTest t;
			t.chi2Mono = atof(f[1].c_str()); t.chi2Stereo = atof(f[2].c_str());
			t.requirePositiveDepth = atoi(f[3].c_str()) != 0; t.reinclude = atoi(f[4].c_str()) != 0;
			const cuba::OutlierCounts c = cuba::classifyEdges(*opt, t);
			printf(", \"counts\": [%zu, %zu, %zu, %zu]", c.includedMono, c.includedStereo, c.excluded, c.reincluded);
			printLevels(*opt, st);
		}
		else if (f[0] == "levels") printLevels(*opt, st);
		else { fprintf(stderr, "unknown op %s\n", op.c_str()); return 2; }
		printf("}");
	}
	printf("]}\n");
	// classifyEdges() before any optimize() is a logic error
	{
		Storage st2;
		auto fresh = readGraph(argv[1], st2);
		bool threw = false;
		try { cuba::classifyEdges(*fresh, cuba::OutlierTest()); } catch (const std::logic_error&) { threw = true; }
		if (!threw) { fprintf(stderr, "classifyEdges before optimize() did not throw std::logic_error\n"); return 3; }
	}
	FILE* fo = fopen(argv[3], "wb");
	if (!fo) return 2;
	for (auto& v : st.poses) fwrite(v->q.coeffs().data(), sizeof(double), 4, fo);
	for (auto& v : st.poses) fwrite(v->t.data(), sizeof(double), 3, fo);
	for (auto& v : st.landmarks) fwrite(v->Xw.data(), sizeof(double), 3, fo);
	fclose(fo);
	return 0;
}
