// cuba_math.cuh -- per-edge / per-vertex arithmetic of the LM hot path, shared by every kernel, and the LM rules (lm::).
//
// Everything here is __host__ __device__ so that tests/test_host_math.py can compile the very same
// functions with g++ and check them against the oracle without a GPU.
//
// Reference behaviour restated (paths relative to the reference checkout; no code copied):
//   projection            src/cuda_block_solver.cu:245-290
//   Jacobians             cu:292-415   (sign convention: d(meas - proj)/dx, SURVEY fact 9)
//   robust kernels        cu:692-727
//   3x3 adjugate inverse  cu:417-452
//   SE(3) exp update      cu:454-592
#pragma once

#include <math.h>

#if defined(__CUDACC__)
#define CUBA_HD __host__ __device__ __forceinline__
#else
#define CUBA_HD inline
#endif

namespace cuba_b200 {

enum { RK_NONE = 0, RK_HUBER = 1, RK_TUKEY = 2 };

template <typename T> CUBA_HD T t_sqrt(T x);
template <> CUBA_HD double t_sqrt<double>(double x) { return sqrt(x); }
template <> CUBA_HD float t_sqrt<float>(float x) { return sqrtf(x); }
template <typename T> CUBA_HD T t_sin(T x);
template <> CUBA_HD double t_sin<double>(double x) { return sin(x); }
template <> CUBA_HD float t_sin<float>(float x) { return sinf(x); }
template <typename T> CUBA_HD T t_cos(T x);
template <> CUBA_HD double t_cos<double>(double x) { return cos(x); }
template <> CUBA_HD float t_cos<float>(float x) { return cosf(x); }

// Xc = R(q) X, quaternion stored x,y,z,w.  Two cross products, like the reference (cu:245-260),
// so that the residuals agree to the last bits.
template <typename T>
CUBA_HD void rotate(const T q[4], const T X[3], T Xc[3])
{
	T a0 = q[1] * X[2] - q[2] * X[1];
	T a1 = q[2] * X[0] - q[0] * X[2];
	T a2 = q[0] * X[1] - q[1] * X[0];
	a0 += a0; a1 += a1; a2 += a2;
	const T b0 = q[1] * a2 - q[2] * a1;
	const T b1 = q[2] * a0 - q[0] * a2;
	const T b2 = q[0] * a1 - q[1] * a0;
	Xc[0] = X[0] + q[3] * a0 + b0;
	Xc[1] = X[1] + q[3] * a1 + b1;
	Xc[2] = X[2] + q[3] * a2 + b2;
}

// rho(e) and rho'(e), e = omega * |r|^2  (cu:692-727)
template <typename T>
CUBA_HD void robust(int type, T delta, T e, T& rho, T& drho)
{
	const T d2 = delta * delta;
	if (type == RK_HUBER) {
		if (e <= d2) { rho = e; drho = T(1); }
		else { const T s = t_sqrt(e); rho = 2 * s * delta - d2; drho = delta / s; }
	} else if (type == RK_TUKEY) {
		const T maxv = (T(1) / 3) * d2;
		if (e <= d2) { const T u = 1 - e / d2; rho = maxv * (1 - u * u * u); drho = u * u; }
		else { rho = maxv; drho = T(0); }
	} else { rho = e; drho = T(1); }
}

// Residual of one edge.  r[2] = 0 for monocular edges.  Returns Xc too (needed by the Jacobians).
// cam = fx,fy,cx,cy,bf.
template <typename T>
CUBA_HD void edge_residual(const T q[4], const T t[3], const T cam[5], const T Xw[3], const T m[3], bool stereo,
	T Xc[3], T r[3])
{
	rotate(q, Xw, Xc);
	Xc[0] += t[0]; Xc[1] += t[1]; Xc[2] += t[2];
	const T invZ = 1 / Xc[2];
	const T u = cam[0] * invZ * Xc[0] + cam[2];
	const T v = cam[1] * invZ * Xc[1] + cam[3];
	r[0] = u - m[0];
	r[1] = v - m[1];
	r[2] = stereo ? ((u - cam[4] * invZ) - m[2]) : T(0);
}

// Jacobians of one edge at camera-frame point Xc.  JP[m][l] (3x6: rotation then translation),
// JL[m][n] (3x3); row 2 is zero for monocular edges so one code path serves both edge types.
template <typename T>
CUBA_HD void edge_jacobians(const T q[4], const T cam[5], const T Xc[3], bool stereo, T JP[3][6], T JL[3][3])
{
	const T x = q[0], y = q[1], z = q[2], w = q[3];
	const T tx = 2 * x, ty = 2 * y, tz = 2 * z;
	const T twx = tx * w, twy = ty * w, twz = tz * w;
	const T txx = tx * x, txy = ty * x, txz = tz * x;
	const T tyy = ty * y, tyz = tz * y, tzz = tz * z;
	const T R00 = 1 - (tyy + tzz), R01 = txy - twz, R02 = txz + twy;
	const T R10 = txy + twz, R11 = 1 - (txx + tzz), R12 = tyz - twx;
	const T R20 = txz - twy, R21 = tyz + twx, R22 = 1 - (txx + tyy);

	const T invZ = 1 / Xc[2];
	const T xn = invZ * Xc[0], yn = invZ * Xc[1];
	const T fu = cam[0], fv = cam[1];
	const T fuZ = fu * invZ, fvZ = fv * invZ;

	JL[0][0] = -fuZ * (R00 - xn * R20); JL[0][1] = -fuZ * (R01 - xn * R21); JL[0][2] = -fuZ * (R02 - xn * R22);
	JL[1][0] = -fvZ * (R10 - yn * R20); JL[1][1] = -fvZ * (R11 - yn * R21); JL[1][2] = -fvZ * (R12 - yn * R22);

	JP[0][0] = fu * xn * yn;       JP[0][1] = -fu * (1 + xn * xn); JP[0][2] = fu * yn;
	JP[0][3] = -fuZ;               JP[0][4] = T(0);                JP[0][5] = fuZ * xn;
	JP[1][0] = fv * (1 + yn * yn); JP[1][1] = -fv * xn * yn;       JP[1][2] = -fv * xn;
	JP[1][3] = T(0);               JP[1][4] = -fvZ;                JP[1][5] = fvZ * yn;

	if (stereo) {
		const T bZZ = cam[4] * invZ * invZ;   // bf / Z^2
		JL[2][0] = JL[0][0] - bZZ * R20; JL[2][1] = JL[0][1] - bZZ * R21; JL[2][2] = JL[0][2] - bZZ * R22;
		JP[2][0] = JP[0][0] - bZZ * Xc[1]; JP[2][1] = JP[0][1] + bZZ * Xc[0]; JP[2][2] = JP[0][2];
		JP[2][3] = JP[0][3];               JP[2][4] = T(0);                   JP[2][5] = JP[0][5] - bZZ;
	} else {
#pragma unroll
		for (int i = 0; i < 3; i++) JL[2][i] = T(0);
#pragma unroll
		for (int i = 0; i < 6; i++) JP[2][i] = T(0);
	}
}

// closed-form inverse of a symmetric 3x3 given by its 6 unique entries (cu:417-452, same formula order)
template <typename T>
CUBA_HD void sym3_inverse(T A00, T A01, T A02, T A11, T A12, T A22, T B[6] /* 00,01,02,11,12,22 */)
{
	const T det = A00 * A11 * A22 + A01 * A12 * A02 + A02 * A01 * A12 - A00 * A12 * A12 - A02 * A11 * A02 - A01 * A01 * A22;
	const T id = 1 / det;
	B[0] = id * (A11 * A22 - A12 * A12);
	B[1] = id * (A02 * A12 - A01 * A22);
	B[2] = id * (A01 * A12 - A02 * A11);
	B[3] = id * (A00 * A22 - A02 * A02);
	B[4] = id * (A02 * A01 - A00 * A12);
	B[5] = id * (A00 * A11 - A01 * A01);
}

// In-place inverse of a symmetric positive definite NxN (column-major) via Cholesky; returns false when
// a pivot is not positive.  N = 6: the block-Jacobi preconditioner of the PCG and the pose solves; N = 7: the Sim(3) solve.
template <int N, typename T>
CUBA_HD bool spd_inverse(T A[N * N])
{
	T L[N * N];
#pragma unroll
	for (int i = 0; i < N * N; i++) L[i] = T(0);
	for (int j = 0; j < N; j++) {
		T d = A[j * N + j];
		for (int k = 0; k < j; k++) d -= L[k * N + j] * L[k * N + j];
		if (!(d > T(0))) return false;
		d = t_sqrt(d);
		L[j * N + j] = d;
		const T id = 1 / d;
		for (int i = j + 1; i < N; i++) {
			T s = A[j * N + i];
			for (int k = 0; k < j; k++) s -= L[k * N + i] * L[k * N + j];
			L[j * N + i] = s * id;
		}
	}
	// invert L (lower) into Li
	T Li[N * N];
#pragma unroll
	for (int i = 0; i < N * N; i++) Li[i] = T(0);
	for (int j = 0; j < N; j++) {
		Li[j * N + j] = 1 / L[j * N + j];
		for (int i = j + 1; i < N; i++) {
			T s = T(0);
			for (int k = j; k < i; k++) s -= L[k * N + i] * Li[j * N + k];
			Li[j * N + i] = s / L[i * N + i];
		}
	}
	// A^-1 = Li^T Li
	for (int j = 0; j < N; j++)
		for (int i = 0; i <= j; i++) {
			T s = T(0);
			for (int k = j; k < N; k++) s += Li[i * N + k] * Li[j * N + k];
			A[j * N + i] = s; A[i * N + j] = s;
		}
	return true;
}
template <typename T>
CUBA_HD bool spd6_inverse(T A[36]) { return spd_inverse<6, T>(A); }

// ---- the Levenberg-Marquardt rules of Engine::optimize (reference src/cuda_bundle_adjustment.cpp:793-857), which the batched
// kernels' loop (cuba_lm_batch.cuh) follows too.  A small system of N unknowns is packed as sys[0 .. N(N+1)/2): the upper triangle
// (column n, row l <= n at n (n+1)/2 + l), then b = sys[N(N+1)/2 ..]; the step x solves (H + lambda I) x = b.
namespace lm {

constexpr int MAX_TRIALS = 10;

// lambda of the first iteration: tau times the largest diagonal entry
CUBA_HD double initial_lambda(double maxDiagonal)
{
	const double tau = 1e-5;
	return tau * maxDiagonal;
}

// the largest diagonal entry of a packed system, starting from 0 (k_max_diagonal)
template <int N>
CUBA_HD double max_diagonal(const double* sys)
{
	double md = 0;
#pragma unroll
	for (int d = 0; d < N; d++) { const double v = sys[d * (d + 1) / 2 + d]; md = v > md ? v : md; }
	return md;
}

// the damped solve of a packed system (k_solve_poses_only): x = 0 when the Cholesky of H + lambda I fails
template <int N>
CUBA_HD void damped_solve(const double* sys, double lambda, double x[N])
{
	double M[N * N];
	for (int e = 0; e < N * N; e++) {
		const int cn = e / N, l = e - N * cn;
		const int lo = l < cn ? l : cn, hi = l < cn ? cn : l;
		M[e] = sys[hi * (hi + 1) / 2 + lo] + ((e % (N + 1)) == 0 ? lambda : 0.0);
	}
	if (!spd_inverse<N>(M)) {
		for (int i = 0; i < N; i++) x[i] = 0;
	} else {
		for (int r = 0; r < N; r++) {
			double sum = 0;
			for (int c = 0; c < N; c++) sum += M[c * N + r] * sys[N * (N + 1) / 2 + c];
			x[r] = sum;
		}
	}
}

// the predicted decrease x^T (lambda x + b) of a step
template <int N>
CUBA_HD double predicted_decrease(const double* sys, double lambda, const double x[N])
{
	double sc = 0;
	for (int i = 0; i < N; i++) sc += x[i] * (lambda * x[i] + sys[N * (N + 1) / 2 + i]);
	return sc;
}

// the gain ratio of a trial that takes chi2 from F to Fhat; a NaN ratio rejects the trial
CUBA_HD double gain_ratio(double F, double Fhat, double predicted)
{
	const double scale = predicted + 1e-3;
	double rho = (F - Fhat) / scale;
	if (!(rho == rho)) rho = -1;
	return rho;
}

// the lambda / nu update a trial's gain ratio implies; returns whether the trial is accepted
CUBA_HD bool update_damping(double rho, double& lambda, double& nu)
{
	if (rho > 0) {
		const double x = 2 * rho - 1;
		lambda *= fmax(1. / 3, fmin(1 - x * x * x, 2. / 3));
		nu = 2;
		return true;
	}
	lambda *= nu; nu *= 2;
	return false;
}

// the end of the iterations: every trial of the iteration rejected, no decrease, or lambda no longer finite
CUBA_HD bool stop(int rejected, double rho, double lambda)
{
	return rejected == MAX_TRIALS || rho <= 0 || !isfinite(lambda);
}

}  // namespace lm

// pose <- Exp([omega;upsilon]) * pose  (cu:551-592): Rodrigues with the theta<1e-5 Taylor branch,
// R->quaternion by the trace method (cu:492-521), normalisation with w>=0 (cu:531-539).
// In fp32, a2 = (1 - cos th) / th^2 cancels to nothing between th = 1e-5 and ~3e-4 (V then loses its [w]x upsilon term, an error
// of th/2 |upsilon|), so the float instantiation uses a2 = 1/2 (sin(th/2) / (th/2))^2 and the series of a3 below th = 0.5.  The
// double instantiation keeps the reference's formulas (its cancellation costs at most 1.1e-11 |upsilon|).
template <typename T>
CUBA_HD void se3_coefficients(T theta, T& a1, T& a2, T& a3)
{
	if (theta < T(0.00001)) { a1 = T(1); a2 = T(0.5); a3 = T(1) / 6; }
	else {
		a1 = t_sin(theta) / theta;
		a2 = (1 - t_cos(theta)) / (theta * theta);
		a3 = (theta - t_sin(theta)) / (theta * theta * theta);
	}
}
template <>
CUBA_HD void se3_coefficients<float>(float theta, float& a1, float& a2, float& a3)
{
	if (theta < 0.00001f) { a1 = 1.f; a2 = 0.5f; a3 = 1.f / 6; return; }
	a1 = sinf(theta) / theta;
	const float h = 0.5f * theta, s = sinf(h) / h;
	a2 = 0.5f * s * s;
	const float t2 = theta * theta;
	// (th - sin th) / th^3 = 1/6 - th^2/120 + th^4/5040 - th^6/362880 + ..., truncation below 1e-10 at th = 0.5
	a3 = theta < 0.5f ? (1.f / 6) - t2 * ((1.f / 120) - t2 * ((1.f / 5040) - t2 * (1.f / 362880))) : (theta - sinf(theta)) / (t2 * theta);
}

template <typename T>
CUBA_HD void se3_update(const T upd[6], T q[4], T t[3])
{
	const T wx = upd[0], wy = upd[1], wz = upd[2];
	const T theta = t_sqrt(wx * wx + wy * wy + wz * wz);
	T a1, a2, a3;
	se3_coefficients(theta, a1, a2, a3);
	// O1 = [w]x, O2 = [w]x^2 ; M(i,j) row i col j
	const T O1[3][3] = { { T(0), -wz, wy }, { wz, T(0), -wx }, { -wy, wx, T(0) } };
	const T xx = wx * wx, yy = wy * wy, zz = wz * wz, xy = wx * wy, yz = wy * wz, zx = wz * wx;
	const T O2[3][3] = { { -yy - zz, xy, zx }, { xy, -zz - xx, yz }, { zx, yz, -xx - yy } };
	T R[3][3], V[3][3];
#pragma unroll
	for (int i = 0; i < 3; i++)
#pragma unroll
		for (int j = 0; j < 3; j++) {
			const T I = (i == j) ? T(1) : T(0);
			R[i][j] = I + a1 * O1[i][j] + a2 * O2[i][j];
			V[i][j] = I + a2 * O1[i][j] + a3 * O2[i][j];
		}
	T eq[4];
	T tr = R[0][0] + R[1][1] + R[2][2];
	if (tr > T(0)) {
		tr = t_sqrt(tr + 1);
		eq[3] = T(0.5) * tr; tr = T(0.5) / tr;
		eq[0] = (R[2][1] - R[1][2]) * tr; eq[1] = (R[0][2] - R[2][0]) * tr; eq[2] = (R[1][0] - R[0][1]) * tr;
	} else {
		int i = 0;
		if (R[1][1] > R[0][0]) i = 1;
		if (R[2][2] > R[i][i]) i = 2;
		const int j = (i + 1) % 3, k = (j + 1) % 3;
		tr = t_sqrt(R[i][i] - R[j][j] - R[k][k] + 1);
		eq[i] = T(0.5) * tr; tr = T(0.5) / tr;
		eq[3] = (R[k][j] - R[j][k]) * tr; eq[j] = (R[j][i] + R[i][j]) * tr; eq[k] = (R[k][i] + R[i][k]) * tr;
	}
	T et[3];
#pragma unroll
	for (int i = 0; i < 3; i++) et[i] = V[i][0] * upd[3] + V[i][1] * upd[4] + V[i][2] * upd[5];
	T u[3];
	rotate(eq, t, u);
#pragma unroll
	for (int i = 0; i < 3; i++) t[i] = et[i] + u[i];
	T r[4];
	r[3] = eq[3] * q[3] - eq[0] * q[0] - eq[1] * q[1] - eq[2] * q[2];
	r[0] = eq[3] * q[0] + eq[0] * q[3] + eq[1] * q[2] - eq[2] * q[1];
	r[1] = eq[3] * q[1] + eq[1] * q[3] + eq[2] * q[0] - eq[0] * q[2];
	r[2] = eq[3] * q[2] + eq[2] * q[3] + eq[0] * q[1] - eq[1] * q[0];
	T invn = 1 / t_sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3]);
	if (r[3] < T(0)) invn = -invn;
#pragma unroll
	for (int i = 0; i < 4; i++) q[i] = invn * r[i];
}

// ---- Sim(3): S = (R(q), t, s), S X = s R X + t (cuba_sim3_batch.cuh); double precision only ----

// W = int_0^1 e^(sigma u) exp(u [w]x) du = A I + B [w]x + C [w]x^2, theta = |w|.  The closed forms (A = expm1(sigma) / sigma and
// B, C below) cancel as theta and / or sigma go to 0, so inside |(sigma, theta)| <= 1 W is summed as its series: W = sum_n
// Omega^n / (n+1)!, Omega = sigma I + [w]x, with Omega^n = p I + q [w]x + r [w]x^2 by [w]x^3 = -theta^2 [w]x.  Twenty terms leave a
// truncation below 1/21! there.  Outside, with es = e^sigma, s1 = sin(theta) / theta and h2 = (1 - cos theta) / theta^2 =
// (sin(theta/2) / (theta/2))^2 / 2 (neither cancels):
//   B = (sigma es s1 - expm1(sigma) + es theta^2 h2) / (sigma^2 + theta^2)
//   C = (A - ((es cos(theta) - 1) sigma + es sin(theta) theta) / (sigma^2 + theta^2)) / theta^2    theta >= 1/2
//   C = (es sigma^2 h2 + expm1(sigma) - sigma es s1) / (sigma (sigma^2 + theta^2))                  theta < 1/2 (so |sigma| > 0.86)
CUBA_HD void sim3_coefficients(double sigma, double theta, double& A, double& B, double& C)
{
	const double th2 = theta * theta, c = sigma * sigma + th2;
	if (c <= 1) {
		double p = 1, q = 0, r = 0, f = 1;
		A = 1; B = 0; C = 0;
		for (int n = 1; n <= 20; n++) {
			const double pn = sigma * p, qn = sigma * q + p - th2 * r, rn = sigma * r + q;
			p = pn; q = qn; r = rn;
			f /= (n + 1);
			A += f * p; B += f * q; C += f * r;
		}
		return;
	}
	const double es = exp(sigma), em1 = expm1(sigma);
	const double h = 0.5 * theta, sh = theta > 0 ? sin(h) / h : 1.0;
	const double s1 = theta > 0 ? sin(theta) / theta : 1.0, h2 = 0.5 * sh * sh;
	A = sigma != 0 ? em1 / sigma : 1.0;
	B = (sigma * es * s1 - em1 + es * th2 * h2) / c;
	if (theta >= 0.5) C = (A - ((em1 - es * th2 * h2) * sigma + es * s1 * th2) / c) / th2;
	else C = (es * sigma * sigma * h2 + em1 - sigma * es * s1) / (sigma * c);
}

// S <- Exp(xi) S, xi = (omega, upsilon, sigma) (g2o's VertexSim3Expmap::oplusImpl): R <- Rodrigues(omega) R, t <- e^sigma
// Rodrigues(omega) t + W upsilon, s <- e^sigma s.  The rotation and its quaternion are se3_update's (with upsilon = 0), so with
// sigma = 0 this is se3_update up to the rounding of W = V.  sigma = 0 leaves s bit for bit.
CUBA_HD void sim3_update(const double upd[7], double q[4], double t[3], double& s)
{
	const double w[3] = { upd[0], upd[1], upd[2] }, v[3] = { upd[3], upd[4], upd[5] }, sigma = upd[6];
	double A, B, C;
	sim3_coefficients(sigma, sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]), A, B, C);
	const double wv[3] = { w[1] * v[2] - w[2] * v[1], w[2] * v[0] - w[0] * v[2], w[0] * v[1] - w[1] * v[0] };
	const double wwv[3] = { w[1] * wv[2] - w[2] * wv[1], w[2] * wv[0] - w[0] * wv[2], w[0] * wv[1] - w[1] * wv[0] };
	const double es = exp(sigma);
	for (int i = 0; i < 3; i++) t[i] *= es;
	const double rot[6] = { w[0], w[1], w[2], 0.0, 0.0, 0.0 };
	se3_update(rot, q, t);
	for (int i = 0; i < 3; i++) t[i] += A * v[i] + B * wv[i] + C * wwv[i];
	s *= es;
}

// Y = S X = s R(q) X + t
CUBA_HD void sim3_map(const double q[4], const double t[3], double s, const double X[3], double Y[3])
{
	rotate(q, X, Y);
	for (int i = 0; i < 3; i++) Y[i] = s * Y[i] + t[i];
}

// Z = S^-1 X = R(q)^T (X - t) / s
CUBA_HD void sim3_inverse_map(const double q[4], const double t[3], double s, const double X[3], double Z[3])
{
	const double qc[4] = { -q[0], -q[1], -q[2], q[3] }, d[3] = { X[0] - t[0], X[1] - t[1], X[2] - t[2] };
	rotate(qc, d, Z);
	for (int i = 0; i < 3; i++) Z[i] /= s;
}

// r = pi(P) - obs, pi(P) = (fx P.x / P.z + cx, fy P.y / P.z + cy), cam = fx, fy, cx, cy (the projection of edge_residual)
CUBA_HD void sim3_project(const double cam[4], const double P[3], const double obs[2], double r[2])
{
	const double invZ = 1 / P[2];
	r[0] = cam[0] * invZ * P[0] + cam[2] - obs[0];
	r[1] = cam[1] * invZ * P[1] + cam[3] - obs[1];
}

// d pi / dP (2x3)
CUBA_HD void sim3_project_jacobian(const double cam[4], const double P[3], double Jp[2][3])
{
	const double invZ = 1 / P[2];
	Jp[0][0] = cam[0] * invZ; Jp[0][1] = 0;               Jp[0][2] = -cam[0] * P[0] * invZ * invZ;
	Jp[1][0] = 0;             Jp[1][1] = cam[1] * invZ; Jp[1][2] = -cam[1] * P[1] * invZ * invZ;
}

// e12 of a matched pair: r = pi1(S X2) - obs1; Y = S X2 is returned for the Jacobian
CUBA_HD void sim3_residual12(const double q[4], const double t[3], double s, const double cam1[4], const double X2[3], const double obs1[2],
	double Y[3], double r[2])
{
	sim3_map(q, t, s, X2, Y);
	sim3_project(cam1, Y, obs1, r);
}

// e21 of a matched pair: r = pi2(S^-1 X1) - obs2; Z = S^-1 X1 is returned for the Jacobian
CUBA_HD void sim3_residual21(const double q[4], const double t[3], double s, const double cam2[4], const double X1[3], const double obs2[2],
	double Z[3], double r[2])
{
	sim3_inverse_map(q, t, s, X1, Z);
	sim3_project(cam2, Z, obs2, r);
}

// dr/dxi of e12 for the update Exp(xi) S (2x7, columns omega, upsilon, sigma): d pi1 / dY [-[Y]x, I, Y]
CUBA_HD void sim3_jacobian12(const double cam1[4], const double Y[3], double J[2][7])
{
	double Jp[2][3];
	sim3_project_jacobian(cam1, Y, Jp);
	for (int m = 0; m < 2; m++) {
		const double* a = Jp[m];
		// row m of -Jp [Y]x is Y x a
		J[m][0] = Y[1] * a[2] - Y[2] * a[1]; J[m][1] = Y[2] * a[0] - Y[0] * a[2]; J[m][2] = Y[0] * a[1] - Y[1] * a[0];
		J[m][3] = a[0]; J[m][4] = a[1]; J[m][5] = a[2];
		J[m][6] = a[0] * Y[0] + a[1] * Y[1] + a[2] * Y[2];
	}
}

// dr/dxi of e21 (2x7): d pi2 / dZ (1/s) R^T [[X1]x, -I, -X1]
CUBA_HD void sim3_jacobian21(const double q[4], double s, const double cam2[4], const double X1[3], const double Z[3], double J[2][7])
{
	double Jp[2][3];
	sim3_project_jacobian(cam2, Z, Jp);
	for (int m = 0; m < 2; m++) {
		// row m of M = Jp R^T / s is (R Jp[m]) / s
		double a[3];
		rotate(q, Jp[m], a);
		for (int i = 0; i < 3; i++) a[i] /= s;
		// row m of M [X1]x is a x X1
		J[m][0] = a[1] * X1[2] - a[2] * X1[1]; J[m][1] = a[2] * X1[0] - a[0] * X1[2]; J[m][2] = a[0] * X1[1] - a[1] * X1[0];
		J[m][3] = -a[0]; J[m][4] = -a[1]; J[m][5] = -a[2];
		J[m][6] = -(a[0] * X1[0] + a[1] * X1[1] + a[2] * X1[2]);
	}
}

#if defined(__CUDACC__)
// D = A B + D on the fp64 tensor pipe, one 8x8x4 product per warp: lane l holds A(l/4, l%4), B(l%4, l/4) and
// D(l/4, 2 (l%4)) / D(l/4, 2 (l%4) + 1)
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b)
{
	asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
#endif

}  // namespace cuba_b200
