// solver_driver.cpp -- TEST DRIVER for the linear solver of the drop-in class (include/cuba_b200_solver.h).  Executes a ';'-separated
// op list on a .cubagraph and prints one JSON object; tests/test_dense_solver_dropin.py runs the same steps on the Python Engine.
//   solver:pcg|dense | query (the stored choice, no GPU needed) | kernel:none|huber | init | opt:N | classify:CHI2MONO:CHI2STEREO
//   tryopt:N (optimize(N), reporting whether it threw std::runtime_error instead of stopping)
// The estimate after the last op is written to the dump file (q, t of every pose, Xw of every landmark, file order).
#include <cmath>
#include <sstream>
#include <stdexcept>

#include <cuba_b200.h>
#include <cuba_b200_levels.h>
#include <cuba_b200_solver.h>

#include "../../samples/cubagraph_reader.h"

int main(int argc, char** argv)
{
	if (argc < 4) { fprintf(stderr, "usage: solver_driver graph.cubagraph ops dump.bin\n"); return 2; }
	Storage st;
	auto opt = readGraph(argv[1], st);
	std::stringstream ss(argv[2]);
	std::string op;
	printf("{\"steps\": [");
	bool first = true;
	bool ran = false;
	while (std::getline(ss, op, ';')) {
		if (op.empty()) continue;
		std::vector<std::string> f;
		{ std::stringstream s2(op); std::string x; while (std::getline(s2, x, ':')) f.push_back(x); }
		printf("%s{\"op\": \"%s\"", first ? "" : ", ", op.c_str());
		first = false;
		if (f[0] == "solver") cuba::setLinearSolver(*opt, f[1] == "dense" ? cuba::LinearSolverType::DENSE_CHOLESKY : cuba::LinearSolverType::PCG);
		else if (f[0] == "query") printf(", \"solver\": %d", cuba::linearSolver(*opt) == cuba::LinearSolverType::DENSE_CHOLESKY ? 1 : 0);
		else if (f[0] == "kernel") {
			const bool huber = f[1] == "huber";
			opt->setRobustKernels(huber ? cuba::RobustKernelType::HUBER : cuba::RobustKernelType::NONE, huber ? std::sqrt(5.991) : 0.0, cuba::EdgeType::MONOCULAR);
			opt->setRobustKernels(huber ? cuba::RobustKernelType::HUBER : cuba::RobustKernelType::NONE, huber ? std::sqrt(7.815) : 0.0, cuba::EdgeType::STEREO);
		}
		else if (f[0] == "init") opt->initialize();
		else if (f[0] == "opt") {
			const size_t before = opt->batchStatistics().size();
			opt->optimize(atoi(f[1].c_str()));
			ran = true;
			const auto& s = opt->batchStatistics();
			printf(", \"chi2\": [");
			for (size_t i = before; i < s.size(); i++) printf("%s%.17g", i > before ? ", " : "", s[i].chi2);
			printf("]");
		}
		else if (f[0] == "tryopt") {
			bool threw = false;
			try { opt->optimize(atoi(f[1].c_str())); ran = true; } catch (const std::runtime_error&) { threw = true; }
			printf(", \"threw\": %s", threw ? "true" : "false");
		}
		else if (f[0] == "classify") {
			cuba::OutlierTest t;
			t.chi2Mono = atof(f[1].c_str()); t.chi2Stereo = atof(f[2].c_str());
			const cuba::OutlierCounts c = cuba::classifyEdges(*opt, t);
			printf(", \"counts\": [%zu, %zu, %zu, %zu]", c.includedMono, c.includedStereo, c.excluded, c.reincluded);
		}
		else { fprintf(stderr, "unknown op %s\n", op.c_str()); return 2; }
		printf("}");
	}
	printf("]}\n");
	if (!ran) return 0;
	FILE* fo = fopen(argv[3], "wb");
	if (!fo) return 2;
	for (auto& v : st.poses) fwrite(v->q.coeffs().data(), sizeof(double), 4, fo);
	for (auto& v : st.poses) fwrite(v->t.data(), sizeof(double), 3, fo);
	for (auto& v : st.landmarks) fwrite(v->Xw.data(), sizeof(double), 3, fo);
	fclose(fo);
	return 0;
}
