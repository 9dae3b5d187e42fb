// math_driver.cpp -- TEST DRIVER for the per-edge primitives of csrc/cuba_math.cuh, compiled by the host compiler from the very
// header the kernels include.  tests/test_host_math.py feeds it records on stdin and checks the outputs against numpy restatements.
//   math_driver float|double se3|robust|edge|sym3|spd6  <  records (whitespace-separated numbers, read as double, narrowed to T)
// One output line per record, every value printed as a double with 17 significant digits:
//   se3     in: upd[6] q[4] t[3]                         out: q[4] t[3]
//   robust  in: type delta e                             out: rho drho
//   edge    in: q[4] t[3] cam[5] Xw[3] m[3] stereo       out: Xc[3] r[3] JP[3][6] JL[3][3] (row-major)
//   sym3    in: A00 A01 A02 A11 A12 A22                  out: B[6]
//   spd6    in: A[36] (column-major)                     out: ok A^-1[36]
#include <cstdio>
#include <cstring>

#include "cuba_math.cuh"

using namespace cuba_b200;

template <typename T>
static bool rd(T* v, int n)
{
	for (int i = 0; i < n; i++) {
		double d;
		if (scanf("%lf", &d) != 1) return false;
		v[i] = (T)d;
	}
	return true;
}

template <typename T>
static void wr(const T* v, int n, bool last)
{
	for (int i = 0; i < n; i++) printf("%s%.17g", i ? " " : "", (double)v[i]);
	printf(last ? "\n" : " ");
}

template <typename T>
static int run(const char* fn)
{
	if (!strcmp(fn, "se3")) {
		T u[6], q[4], t[3];
		while (rd(u, 6) && rd(q, 4) && rd(t, 3)) { se3_update(u, q, t); wr(q, 4, false); wr(t, 3, true); }
	} else if (!strcmp(fn, "robust")) {
		T v[3];
		while (rd(v, 3)) { T rho, drho; robust((int)v[0], v[1], v[2], rho, drho); T o[2] = { rho, drho }; wr(o, 2, true); }
	} else if (!strcmp(fn, "edge")) {
		T q[4], t[3], cam[5], Xw[3], m[3], st[1];
		while (rd(q, 4) && rd(t, 3) && rd(cam, 5) && rd(Xw, 3) && rd(m, 3) && rd(st, 1)) {
			T Xc[3], r[3], JP[3][6], JL[3][3];
			const bool stereo = st[0] != T(0);
			edge_residual(q, t, cam, Xw, m, stereo, Xc, r);
			edge_jacobians(q, cam, Xc, stereo, JP, JL);
			wr(Xc, 3, false); wr(r, 3, false); wr(&JP[0][0], 18, false); wr(&JL[0][0], 9, true);
		}
	} else if (!strcmp(fn, "sym3")) {
		T A[6], B[6];
		while (rd(A, 6)) { sym3_inverse(A[0], A[1], A[2], A[3], A[4], A[5], B); wr(B, 6, true); }
	} else if (!strcmp(fn, "spd6")) {
		T A[36];
		while (rd(A, 36)) { const T ok = spd6_inverse(A) ? T(1) : T(0); wr(&ok, 1, false); wr(A, 36, true); }
	} else {
		fprintf(stderr, "unknown function %s\n", fn);
		return 2;
	}
	return 0;
}

int main(int argc, char** argv)
{
	if (argc != 3) { fprintf(stderr, "usage: math_driver float|double se3|robust|edge|sym3|spd6 < records\n"); return 2; }
	if (!strcmp(argv[1], "float")) return run<float>(argv[2]);
	if (!strcmp(argv[1], "double")) return run<double>(argv[2]);
	fprintf(stderr, "unknown type %s\n", argv[1]);
	return 2;
}
