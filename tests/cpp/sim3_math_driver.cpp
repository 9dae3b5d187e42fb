// sim3_math_driver.cpp -- TEST DRIVER for the Sim(3) primitives of csrc/cuba_math.cuh (and spd_inverse<7>), compiled by the host
// compiler from the very header the kernels include.  tests/test_sim3_batch.py feeds it records on stdin.
//   sim3_math_driver sim3|se3|edge|spd7  <  records (whitespace-separated numbers, read as double)
// One output line per record, every value printed with 17 significant digits:
//   sim3   in: upd[7] q[4] t[3] s                          out: q[4] t[3] s
//   se3    in: upd[6] q[4] t[3]                            out: q[4] t[3]
//   edge   in: q[4] t[3] s cam1[4] cam2[4] X1[3] X2[3] obs1[2] obs2[2]
//          out: r12[2] r21[2] J12[2][7] J21[2][7] (row-major)
//   spd7   in: A[49] (column-major)                        out: ok A^-1[49]
#include <cstdio>
#include <cstring>

#include "cuba_math.cuh"

using namespace cuba_b200;

static bool rd(double* v, int n)
{
	for (int i = 0; i < n; i++)
		if (scanf("%lf", &v[i]) != 1) return false;
	return true;
}

static void wr(const double* v, int n, bool last)
{
	for (int i = 0; i < n; i++) printf("%s%.17g", i ? " " : "", v[i]);
	printf(last ? "\n" : " ");
}

int main(int argc, char** argv)
{
	if (argc != 2) { fprintf(stderr, "usage: sim3_math_driver sim3|se3|edge|spd7 < records\n"); return 2; }
	const char* fn = argv[1];
	if (!strcmp(fn, "sim3")) {
		double u[7], q[4], t[3], s;
		while (rd(u, 7) && rd(q, 4) && rd(t, 3) && rd(&s, 1)) { sim3_update(u, q, t, s); wr(q, 4, false); wr(t, 3, false); wr(&s, 1, true); }
	} else if (!strcmp(fn, "se3")) {
		double u[6], q[4], t[3];
		while (rd(u, 6) && rd(q, 4) && rd(t, 3)) { se3_update(u, q, t); wr(q, 4, false); wr(t, 3, true); }
	} else if (!strcmp(fn, "edge")) {
		double q[4], t[3], s, c1[4], c2[4], X1[3], X2[3], o1[2], o2[2];
		while (rd(q, 4) && rd(t, 3) && rd(&s, 1) && rd(c1, 4) && rd(c2, 4) && rd(X1, 3) && rd(X2, 3) && rd(o1, 2) && rd(o2, 2)) {
			double Y[3], Z[3], r12[2], r21[2], J12[2][7], J21[2][7];
			sim3_residual12(q, t, s, c1, X2, o1, Y, r12);
			sim3_jacobian12(c1, Y, J12);
			sim3_residual21(q, t, s, c2, X1, o2, Z, r21);
			sim3_jacobian21(q, s, c2, X1, Z, J21);
			wr(r12, 2, false); wr(r21, 2, false); wr(&J12[0][0], 14, false); wr(&J21[0][0], 14, true);
		}
	} else if (!strcmp(fn, "spd7")) {
		double A[49];
		while (rd(A, 49)) { const double ok = spd_inverse<7>(A) ? 1.0 : 0.0; wr(&ok, 1, false); wr(A, 49, true); }
	} else {
		fprintf(stderr, "unknown function %s\n", fn);
		return 2;
	}
	return 0;
}
