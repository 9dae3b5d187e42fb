// cuba_math.cuh -- per-edge / per-vertex arithmetic of the LM hot path, shared by every kernel.
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

// In-place inverse of a symmetric positive definite 6x6 (column-major) via Cholesky; returns false when
// a pivot is not positive (block-Jacobi preconditioner of the PCG).
template <typename T>
CUBA_HD bool spd6_inverse(T A[36])
{
	T L[36];
#pragma unroll
	for (int i = 0; i < 36; i++) L[i] = T(0);
	for (int j = 0; j < 6; j++) {
		T d = A[j * 6 + j];
		for (int k = 0; k < j; k++) d -= L[k * 6 + j] * L[k * 6 + j];
		if (!(d > T(0))) return false;
		d = t_sqrt(d);
		L[j * 6 + j] = d;
		const T id = 1 / d;
		for (int i = j + 1; i < 6; i++) {
			T s = A[j * 6 + i];
			for (int k = 0; k < j; k++) s -= L[k * 6 + i] * L[k * 6 + j];
			L[j * 6 + i] = s * id;
		}
	}
	// invert L (lower) into Li
	T Li[36];
#pragma unroll
	for (int i = 0; i < 36; i++) Li[i] = T(0);
	for (int j = 0; j < 6; j++) {
		Li[j * 6 + j] = 1 / L[j * 6 + j];
		for (int i = j + 1; i < 6; i++) {
			T s = T(0);
			for (int k = j; k < i; k++) s -= L[k * 6 + i] * Li[j * 6 + k];
			Li[j * 6 + i] = s / L[i * 6 + i];
		}
	}
	// A^-1 = Li^T Li
	for (int j = 0; j < 6; j++)
		for (int i = 0; i <= j; i++) {
			T s = T(0);
			for (int k = j; k < 6; k++) s += Li[i * 6 + k] * Li[j * 6 + k];
			A[j * 6 + i] = s; A[i * 6 + j] = s;
		}
	return true;
}

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

#if defined(__CUDACC__)
// D = A B + D on the fp64 tensor pipe, one 8x8x4 product per warp: lane l holds A(l/4, l%4), B(l%4, l/4) and
// D(l/4, 2 (l%4)) / D(l/4, 2 (l%4) + 1)
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b)
{
	asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
#endif

}  // namespace cuba_b200
