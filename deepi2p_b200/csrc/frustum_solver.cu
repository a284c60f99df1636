// Batched robust bounded Levenberg-Marquardt solver for the inverse-camera-projection
// ("frustum") registration problem, written for sm_90a (H100).
//
// Replaces FrustumRegistration.solvePGivenK (evaluation/frustum_reg/src/registration.cpp:9-186)
// and the multi-start loop around it (evaluation/registration_lsq.py:127-186).
//
// Execution model (round 2): ONE WARP owns one (cloud, labels, intrinsics, init pose) problem from its
// first evaluation to its final pose; a CTA is a team of 10 warps (two CTAs per SM) that share nothing in the
// steady state -- there is no CTA-wide barrier anywhere in the solve loop.  A pass over the cloud is cut
// into a FIXED sequence of slices (a few rounds of 32 groups x 32 points each); each slice is reduced on
// its own, in a fixed order, and the slice sums are added in slice order.  Because a slice's sum does not
// depend on which warp computed it, warps that have run out of problems (the end-of-kernel tail, small
// batches, the single-problem drop-in call) claim open slices of their CTA-mates' passes through shared
// memory and the results stay bit-identical run to run and independent of who helped.
// The cloud's 32-point groups are dealt round-robin over the rounds, so that every slice carries the same share of
// the exact-path work (a sliced pass is as slow as its heaviest slice).
//
// Per slice a warp culls whole 32-point groups against the frustum with a per-launch box table,
// classifies the points of undecided groups in fp32 with a conservative margin, evaluates the
// maybe-active ones exactly in fp64 (residual, analytic Jacobian, Cauchy corrector) and reduces cost,
// J^T r and J^T J; lane 0 of the owning warp runs the trust-region control flow (Jacobi scaling, LM
// damping, Cholesky of the damped normal matrix, model cost change, box projection, projected Armijo
// line search with cubic interpolation, step acceptance and the tolerance tests) without ever returning
// to the host.  A persistent grid pulls problems from an atomic queue; a second tiny kernel takes the
// per-sample arg-min over inits and builds the 4x4.
//
// Residual definitions: registration_3d.hpp:34-68,105-127 / registration_2d.hpp:34-69,106-129.
// Algorithm text: SURVEY.md Appendix A; oracle/frustum_oracle.cpp is the CPU checker.
#include <cfloat>
#include <cmath>
#include <cstdarg>
#include <cstdlib>

#include "common.cuh"

namespace dib {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// Team shape: warps per CTA (= the help domain: warps that can take slices of each other's passes) x CTAs per SM
// (= problems in flight per SM / warps per CTA).  The register budget decides the product: 20 warps x 32 lanes x 96
// registers for the 4-DoF solver, 14 for 6-DoF (128 registers) and for the f64 record (rings twice as large); shared
// memory (rings + accumulators + per-problem state, ~10.6 KB per 4-DoF warp) is checked below.  An H100 SM has 64 K
// registers and 228 KB of shared memory.  Smaller CTAs leave the SM earlier at the end of a launch (the next launch's
// CTAs start there); 10 x 2 keeps a help domain of 10 warps, which is what a small batch's 10 slices per pass can use.
#ifndef DIB_WARPS_F4
#define DIB_WARPS_F4 10
#endif
#ifndef DIB_WARPS_F6
#define DIB_WARPS_F6 7
#endif
#ifndef DIB_WARPS_D4
#define DIB_WARPS_D4 7
#endif
#ifndef DIB_WARPS_D6
#define DIB_WARPS_D6 5
#endif
#ifndef DIB_CTAS_PER_SM
#define DIB_CTAS_PER_SM 2
#endif
template <typename CT, int P> struct Cfg;
template <> struct Cfg<float, 4> { static constexpr int kWarps = DIB_WARPS_F4; };
template <> struct Cfg<float, 6> { static constexpr int kWarps = DIB_WARPS_F6; };
template <> struct Cfg<double, 4> { static constexpr int kWarps = DIB_WARPS_D4; };
template <> struct Cfg<double, 6> { static constexpr int kWarps = DIB_WARPS_D6; };

struct Cam {
  double fx, fy, cx, cy, W1, H1, hW, hH;
};

// Per-evaluation pose constants, computed once by thread 0 and broadcast through shared memory.
struct PoseConst {
  double R[9];    // rotation applied to the point (first-order I + [a]x when |a|^2 <= DBL_EPSILON)
  double t[3];
  double Jl[9];   // 6-DoF: left Jacobian of SO(3); d(R p)/da = -[R p]x Jl
  double cD, sD;  // 4-DoF: cos/sin used in d q / d ry
  int small;      // first-order branch taken
};

template <int P>
struct NAcc {
  static constexpr int NA = P * (P + 1) / 2;
  static constexpr int N = 1 + P + NA;   // cost, g, packed upper triangle of J^T J
};

__host__ __device__ constexpr int tri(int P, int j, int k) {   // j <= k
  return j * P - j * (j - 1) / 2 + (k - j);
}


// ------------------------------------------------------------------------------------------
// Pose constants.
// ------------------------------------------------------------------------------------------
template <int P>
__device__ __noinline__ void make_pose(const double* x, PoseConst* pc) {
  if (P == 4) {
    const double ry = x[0];
    pc->t[0] = x[1]; pc->t[1] = x[2]; pc->t[2] = x[3];
    double c, s;
    if (ry * ry > DBL_EPSILON) { sincos(ry, &s, &c); pc->cD = c; pc->sD = s; pc->small = 0; }
    else { c = 1.0; s = ry; pc->cD = 1.0; pc->sD = 0.0; pc->small = 1; }
    pc->R[0] = c; pc->R[1] = 0; pc->R[2] = s;
    pc->R[3] = 0; pc->R[4] = 1; pc->R[5] = 0;
    pc->R[6] = -s; pc->R[7] = 0; pc->R[8] = c;
  } else {
    const double ax = x[0], ay = x[1], az = x[2];
    pc->t[0] = x[3]; pc->t[1] = x[4]; pc->t[2] = x[5];
    const double th2 = ax * ax + ay * ay + az * az;
    if (th2 > DBL_EPSILON) {
      const double th = sqrt(th2);
      double s, c;
      sincos(th, &s, &c);
      const double wx = ax / th, wy = ay / th, wz = az / th;
      const double omc = 1.0 - c;
      pc->R[0] = c + wx * wx * omc;      pc->R[1] = wx * wy * omc - wz * s; pc->R[2] = wy * s + wx * wz * omc;
      pc->R[3] = wz * s + wx * wy * omc; pc->R[4] = c + wy * wy * omc;      pc->R[5] = -wx * s + wy * wz * omc;
      pc->R[6] = -wy * s + wx * wz * omc; pc->R[7] = wx * s + wy * wz * omc; pc->R[8] = c + wz * wz * omc;
      // Jl = I + A [a]x + B [a]x^2,  A = (1-cos)/th^2,  B = (th - sin)/th^3   (cancellation-free forms)
      double sh, ch;
      sincos(0.5 * th, &sh, &ch);
      const double q = sh / (0.5 * th);
      const double A = 0.5 * q * q;
      double B;
      if (th < 0.5) {
        const double t2 = th2;
        B = 1.0 / 6.0 + t2 * (-1.0 / 120.0 + t2 * (1.0 / 5040.0 + t2 * (-1.0 / 362880.0 +
            t2 * (1.0 / 39916800.0 + t2 * (-1.0 / 6227020800.0 + t2 * (1.0 / 1307674368000.0))))));
      } else {
        B = (th - s) / (th2 * th);
      }
      // [a]x^2 = a a^T - th2 I
      pc->Jl[0] = 1.0 + B * (ax * ax - th2); pc->Jl[1] = -A * az + B * ax * ay;     pc->Jl[2] = A * ay + B * ax * az;
      pc->Jl[3] = A * az + B * ax * ay;      pc->Jl[4] = 1.0 + B * (ay * ay - th2); pc->Jl[5] = -A * ax + B * ay * az;
      pc->Jl[6] = -A * ay + B * ax * az;     pc->Jl[7] = A * ax + B * ay * az;      pc->Jl[8] = 1.0 + B * (az * az - th2);
      pc->small = 0;
    } else {
      pc->R[0] = 1;   pc->R[1] = -az; pc->R[2] = ay;
      pc->R[3] = az;  pc->R[4] = 1;   pc->R[5] = -ax;
      pc->R[6] = -ay; pc->R[7] = ax;  pc->R[8] = 1;
      for (int i = 0; i < 9; ++i) pc->Jl[i] = (i % 4 == 0) ? 1.0 : 0.0;
      pc->small = 1;
    }
    pc->cD = 0; pc->sD = 0;
  }
}

// ------------------------------------------------------------------------------------------
// Per-point evaluation.  acc = [cost, g[P], packed upper J^T J]; everything weighted by the
// Cauchy corrector w = rho'(s) = 1/(1+s) (CauchyLoss(1.0), registration.cpp:103,121).
// ------------------------------------------------------------------------------------------
// Accumulator view over shared memory: acc[j] is column `lane` of row j ([N][32] doubles per warp).
struct SmemAcc {
  double* base;
  __device__ __forceinline__ double& operator[](int j) const { return base[j * 32]; }
};

template <int P, typename ACC>
__device__ __forceinline__ void rank1(ACC acc, const double* J, double w, double r) {
  const double wr = w * r;
#pragma unroll
  for (int j = 0; j < P; ++j) {
    acc[1 + j] = fma(wr, J[j], acc[1 + j]);
    const double wj = w * J[j];
#pragma unroll
    for (int k = j; k < P; ++k) acc[1 + P + tri(P, j, k)] = fma(wj, J[k], acc[1 + P + tri(P, j, k)]);
  }
}

// Rows of the block Jacobian before robustification.  Returns the number of rows (1 or 3) and
// fills r[] and J[][P]; inactive rows are exactly zero.
template <int P>
__device__ __forceinline__ bool point_rows(double px, double py, double pz, int lab, const Cam& cam,
                                           const PoseConst& pc, double r[3], double J[3][P], int* nrows) {
  constexpr int NR = P - 3;
  const double rx = fma(pc.R[0], px, fma(pc.R[1], py, pc.R[2] * pz));
  const double ry_ = fma(pc.R[3], px, fma(pc.R[4], py, pc.R[5] * pz));
  const double rz = fma(pc.R[6], px, fma(pc.R[7], py, pc.R[8] * pz));
  const double X = rx + pc.t[0], Y = ry_ + pc.t[1], Z = rz + pc.t[2];
  const double iz = 1.0 / Z;
  const double u = fma(cam.fx * X, iz, cam.cx);
  const double v = fma(cam.fy * Y, iz, cam.cy);

  bool any = false;
  double su = 0.0, sv = 0.0, sz = 0.0;   // d r / d u, d r / d v, d r / d Z selectors per row
  if (lab == 0) {
    *nrows = 1;
    const double du_ = u - cam.hW, dv_ = v - cam.hH;
    const double xd = cam.hW - fabs(du_);
    const double yd = cam.hH - fabs(dv_);
    r[0] = 0.0;
    if (Z > 0.0 && xd > 0.0 && yd > 0.0) {
      r[0] = xd + yd;
      su = (du_ < 0.0) ? 1.0 : -1.0;     // -sgn(u - W1/2), sgn(0) = +1
      sv = (dv_ < 0.0) ? 1.0 : -1.0;
      any = true;
    }
  } else {
    *nrows = 3;
    const double a0 = -u, b0 = u - cam.W1;
    const double a1 = -v, b1 = v - cam.H1;
    r[0] = (a0 < 0.0 ? 0.0 : a0) + (b0 < 0.0 ? 0.0 : b0);
    r[1] = (a1 < 0.0 ? 0.0 : a1) + (b1 < 0.0 ? 0.0 : b1);
    r[2] = (-Z < 0.0 ? 0.0 : -Z) * 100.0;
    su = (a0 < 0.0 ? 0.0 : -1.0) + (b0 < 0.0 ? 0.0 : 1.0);
    sv = (a1 < 0.0 ? 0.0 : -1.0) + (b1 < 0.0 ? 0.0 : 1.0);
    sz = (-Z < 0.0) ? 0.0 : -100.0;
    any = (su != 0.0) || (sv != 0.0) || (sz != 0.0);
  }
  if (!any) return false;

  // d q / d rot (NR columns).
  double dX[NR], dY[NR], dZ[NR];
  if (P == 4) {
    dX[0] = fma(-pc.sD, px, pc.cD * pz);
    dY[0] = 0.0;
    dZ[0] = -fma(pc.cD, px, pc.sD * pz);
  } else {
    const double a = pc.small ? px : rx, b = pc.small ? py : ry_, c = pc.small ? pz : rz;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      dX[k] = c * pc.Jl[3 + k] - b * pc.Jl[6 + k];
      dY[k] = a * pc.Jl[6 + k] - c * pc.Jl[k];
      dZ[k] = b * pc.Jl[k] - a * pc.Jl[3 + k];
    }
  }
  const double au = cam.fx * iz, bu = (u - cam.cx) * iz;   // du = au dX - bu dZ
  const double av = cam.fy * iz, bv = (v - cam.cy) * iz;   // dv = av dY - bv dZ
  double dU[P], dV[P];
#pragma unroll
  for (int k = 0; k < NR; ++k) {
    dU[k] = au * dX[k] - bu * dZ[k];
    dV[k] = av * dY[k] - bv * dZ[k];
  }
  dU[NR] = au; dU[NR + 1] = 0.0; dU[NR + 2] = -bu;
  dV[NR] = 0.0; dV[NR + 1] = av; dV[NR + 2] = -bv;
  if (lab == 0) {
#pragma unroll
    for (int j = 0; j < P; ++j) J[0][j] = su * dU[j] + sv * dV[j];
  } else {
#pragma unroll
    for (int j = 0; j < P; ++j) { J[0][j] = su * dU[j]; J[1][j] = sv * dV[j]; }
#pragma unroll
    for (int k = 0; k < NR; ++k) J[2][k] = sz * dZ[k];
    J[2][NR] = 0.0; J[2][NR + 1] = 0.0; J[2][NR + 2] = sz;
  }
  return true;
}

// ------------------------------------------------------------------------------------------
// Branch-free evaluators used by the solver's hot loop.  Batches are homogeneous in the label and
// every lane evaluates two points, so that two independent dependency chains are in flight per
// lane.  `valid == false` (padding lane) and exact-inactive points contribute exactly zero.
// ------------------------------------------------------------------------------------------
template <int P>
struct Proj {
  double X, Y, Z, iz, u, v;
  double dX[P - 3], dY[P - 3], dZ[P - 3];
};

template <int P>
__device__ __forceinline__ void project_point(double px, double py, double pz, bool valid, const Cam& cam,
                                              const PoseConst& pc, Proj<P>& o) {
  constexpr int NR = P - 3;
  if (!valid) { px = 0.0; py = 0.0; pz = 0.0; }
  double rx, ry_, rz;
  if (P == 4) {        // R = Ry(ry): rows (c 0 s), (0 1 0), (-s 0 c); the zero / unit entries are exact, so this is
    rx = fma(pc.R[0], px, pc.R[2] * pz);            // bit-identical to the general form below
    ry_ = py;
    rz = fma(pc.R[6], px, pc.R[8] * pz);
  } else {
    rx = fma(pc.R[0], px, fma(pc.R[1], py, pc.R[2] * pz));
    ry_ = fma(pc.R[3], px, fma(pc.R[4], py, pc.R[5] * pz));
    rz = fma(pc.R[6], px, fma(pc.R[7], py, pc.R[8] * pz));
  }
  o.X = rx + pc.t[0]; o.Y = ry_ + pc.t[1]; o.Z = rz + pc.t[2];
  const double zs = (valid && o.Z != 0.0) ? o.Z : 1.0;     // keeps masked lanes finite
  o.iz = 1.0 / zs;
  o.u = fma(cam.fx * o.X, o.iz, cam.cx);
  o.v = fma(cam.fy * o.Y, o.iz, cam.cy);
  if (P == 4) {
    o.dX[0] = fma(-pc.sD, px, pc.cD * pz);
    o.dY[0] = 0.0;
    o.dZ[0] = -fma(pc.cD, px, pc.sD * pz);
  } else {
    const double a = pc.small ? px : rx, b = pc.small ? py : ry_, c = pc.small ? pz : rz;
#pragma unroll
    for (int k = 0; k < NR; ++k) {
      o.dX[k] = c * pc.Jl[3 + k] - b * pc.Jl[6 + k];
      o.dY[k] = a * pc.Jl[6 + k] - c * pc.Jl[k];
      o.dZ[k] = b * pc.Jl[k] - a * pc.Jl[3 + k];
    }
  }
}

// label 0 ("should be outside", registration_3d.hpp:34-68): one dense row.
template <int P>
struct Out0 {
  double w, r, s1;      // corrector weight (0 if inactive), residual, 1 + s
  double J[P];
};

template <int P>
__device__ __forceinline__ void eval_outside(double px, double py, double pz, bool valid, const Cam& cam,
                                             const PoseConst& pc, Out0<P>& o) {
  constexpr int NR = P - 3;
  Proj<P> q;
  project_point<P>(px, py, pz, valid, cam, pc, q);
  const double du_ = q.u - cam.hW, dv_ = q.v - cam.hH;
  const double xd = cam.hW - fabs(du_), yd = cam.hH - fabs(dv_);
  const bool act = valid && q.Z > 0.0 && xd > 0.0 && yd > 0.0;
  const double su = (du_ < 0.0) ? 1.0 : -1.0;      // -sgn(u - W1/2), sgn(0) = +1
  const double sv = (dv_ < 0.0) ? 1.0 : -1.0;
  o.r = act ? xd + yd : 0.0;
  o.s1 = fma(o.r, o.r, 1.0);
  o.w = act ? 1.0 / o.s1 : 0.0;
  const double au = su * (cam.fx * q.iz), bu = su * ((q.u - cam.cx) * q.iz);
  const double av = sv * (cam.fy * q.iz), bv = sv * ((q.v - cam.cy) * q.iz);
#pragma unroll
  for (int k = 0; k < NR; ++k) {
    double j = au * q.dX[k] - (bu + bv) * q.dZ[k];
    if (P != 4) j = fma(av, q.dY[k], j);
    o.J[k] = j;
  }
  o.J[NR] = au; o.J[NR + 1] = av; o.J[NR + 2] = -(bu + bv);
}

// label 1 ("should be inside", registration_3d.hpp:105-127): three sparse rows
//   JU = su dU (no ty entry), JV = sv dV (no tx entry), JZ = sz dZ (rot and tz entries only).
template <int P>
struct Out1 {
  double w, r0, r1, r2, s1;
  double JU[P], JV[P], JZ[P];
};

template <int P>
__device__ __forceinline__ void eval_inside(double px, double py, double pz, bool valid, const Cam& cam,
                                            const PoseConst& pc, Out1<P>& o) {
  constexpr int NR = P - 3;
  Proj<P> q;
  project_point<P>(px, py, pz, valid, cam, pc, q);
  const double a0 = -q.u, b0 = q.u - cam.W1;
  const double a1 = -q.v, b1 = q.v - cam.H1;
  double su = (a0 < 0.0 ? 0.0 : -1.0) + (b0 < 0.0 ? 0.0 : 1.0);
  double sv = (a1 < 0.0 ? 0.0 : -1.0) + (b1 < 0.0 ? 0.0 : 1.0);
  double sz = (-q.Z < 0.0) ? 0.0 : -100.0;
  o.r0 = (a0 < 0.0 ? 0.0 : a0) + (b0 < 0.0 ? 0.0 : b0);
  o.r1 = (a1 < 0.0 ? 0.0 : a1) + (b1 < 0.0 ? 0.0 : b1);
  o.r2 = (-q.Z < 0.0 ? 0.0 : -q.Z) * 100.0;
  if (!valid) { su = 0.0; sv = 0.0; sz = 0.0; o.r0 = 0.0; o.r1 = 0.0; o.r2 = 0.0; }
  o.s1 = fma(o.r0, o.r0, fma(o.r1, o.r1, fma(o.r2, o.r2, 1.0)));
  o.w = 1.0 / o.s1;
  const double au = su * (cam.fx * q.iz), bu = su * ((q.u - cam.cx) * q.iz);
  const double av = sv * (cam.fy * q.iz), bv = sv * ((q.v - cam.cy) * q.iz);
#pragma unroll
  for (int k = 0; k < NR; ++k) {
    o.JU[k] = au * q.dX[k] - bu * q.dZ[k];
    o.JV[k] = (P == 4) ? -bv * q.dZ[k] : av * q.dY[k] - bv * q.dZ[k];
    o.JZ[k] = sz * q.dZ[k];
  }
  o.JU[NR] = au;  o.JU[NR + 1] = 0.0; o.JU[NR + 2] = -bu;
  o.JV[NR] = 0.0; o.JV[NR + 1] = av;  o.JV[NR + 2] = -bv;
  o.JZ[NR] = 0.0; o.JZ[NR + 1] = 0.0; o.JZ[NR + 2] = sz;
}

// rank-1 update restricted to the entries of J that can be non-zero (compile-time MASK).
template <int P, unsigned MASK, typename ACC>
__device__ __forceinline__ void rank1_masked(ACC acc, const double* J, double w, double r) {
  const double wr = w * r;
#pragma unroll
  for (int j = 0; j < P; ++j) {
    if ((MASK >> j) & 1u) {
      acc[1 + j] = fma(wr, J[j], acc[1 + j]);
      const double wj = w * J[j];
#pragma unroll
      for (int k = j; k < P; ++k)
        if ((MASK >> k) & 1u) acc[1 + P + tri(P, j, k)] = fma(wj, J[k], acc[1 + P + tri(P, j, k)]);
    }
  }
}

template <int P, typename ACC>
__device__ __forceinline__ void accumulate_inside(ACC acc, const Out1<P>& o) {
  constexpr int NR = P - 3;
  constexpr unsigned ROT = (1u << NR) - 1u;
  rank1_masked<P, ROT | (1u << NR) | (1u << (NR + 2)), ACC>(acc, o.JU, o.w, o.r0);
  rank1_masked<P, ROT | (1u << (NR + 1)) | (1u << (NR + 2)), ACC>(acc, o.JV, o.w, o.r1);
  rank1_masked<P, ROT | (1u << (NR + 2)), ACC>(acc, o.JZ, o.w, o.r2);
}

// Running product of (1 + s) kept as mantissa in [1,2) x 2^expo: sum log(1+s) = log(prod) + expo ln 2.
__device__ __forceinline__ void renorm_product(double& prod, int& expo) {
  const int hi = __double2hiint(prod);
  const int e = ((hi >> 20) & 0x7ff) - 1023;
  if (e != 1024) {                       // leave inf / NaN alone so that they propagate
    expo += e;
    prod = __hiloint2double(hi - (e << 20), __double2loint(prod));
  }
}

// ------------------------------------------------------------------------------------------
// Conservative fp32 activity test.  Most points contribute exactly zero to cost, gradient and
// J^T J at a given pose (an "outside" point that projects outside, an "inside" point that
// projects inside).  Each test  u > 0, u < W1, v > 0, v < H1, Z > 0  is, for Z > 0, the sign of
// a linear form in (x, y, z, 1) whose coefficients depend only on the pose and intrinsics:
//     u > 0   <=>  fx X + cx Z        > 0        u < W1  <=>  fx X + (cx - W1) Z < 0
//     v > 0   <=>  fy Y + cy Z        > 0        v < H1  <=>  fy Y + (cy - H1) Z < 0
// The forms are evaluated in fp32 with a per-point error margin m >= 1.6 x the worst-case fp32
// evaluation error (coefficients rounded from fp64, two/three FMAs, inputs possibly rounded from
// fp64).  A point is skipped only if its state is decided by more than m; everything else is
// re-evaluated exactly in fp64, so the sums are those of an all-fp64 evaluation.
// ------------------------------------------------------------------------------------------
struct alignas(16) ClassConst {          // 16-byte rows: one 128-bit shared-memory load each
  float zc[4], al[4], ah[4], bl[4], bh[4];
  float G, G0;
  int enabled;
};

// Warp-collective (all 32 lanes call): lane l < 20 computes coefficient l of the five forms (form l >> 2, column
// l & 3, column 3 = the constant term); the error-margin scales are shuffle reductions (max is exact in any order).
__device__ __forceinline__ void make_class(const PoseConst& pc, const Cam& cam, ClassConst* cc, int lane) {
  const double gamma = 8.0 / 16777216.0;    // 8 * 2^-24
  // the five forms kx X + ky Y + kz Z:  Z;  fx X + cx Z;  fx X + (cx - W1) Z;  fy Y + cy Z;  fy Y + (cy - H1) Z
  const int f = lane >> 2, j = lane & 3;
  double c = 0.0;
  if (lane < 20) {
    const double kx = (f == 1 || f == 2) ? cam.fx : 0.0;
    const double ky = (f >= 3) ? cam.fy : 0.0;
    const double kz = (f == 0) ? 1.0 : (f == 1) ? cam.cx : (f == 2) ? cam.cx - cam.W1 : (f == 3) ? cam.cy : cam.cy - cam.H1;
    const double a0 = (j < 3) ? pc.R[j] : pc.t[0];
    const double a1 = (j < 3) ? pc.R[3 + j] : pc.t[1];
    const double a2 = (j < 3) ? pc.R[6 + j] : pc.t[2];
    c = fma(kx, a0, fma(ky, a1, kz * a2));
  }
  const float cf = (float)c;
  if (lane < 20) cc->zc[lane] = cf;           // zc, al, ah, bl, bh are contiguous float[4]
  double amax = (lane < 20 && j < 3) ? fabs(c) : 0.0;      // largest coefficient of (x, y, z)
  double cmax = (lane < 20 && j == 3) ? fabs(c) : 0.0;     // largest constant term
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    cmax = fmax(cmax, __shfl_xor_sync(0xffffffffu, cmax, o));
  }
  const bool finite = __all_sync(0xffffffffu, isfinite(cf));
  if (lane == 0) {
    cc->G = (float)(gamma * amax * 1.0000002);
    cc->G0 = (float)(gamma * cmax * 1.0000002) + 1e-30f;
    cc->enabled = (finite && isfinite(cc->G) && isfinite(cc->G0)) ? 1 : 0;
  }
}

template <int P>
__device__ __forceinline__ bool maybe_active(float x, float y, float z, int lab, const ClassConst& cc) {
  // branch-free on purpose: the DIB_GPS groups of a step are then classified as one straight-line block that
  // shares the loads of `cc` and interleaves the independent FMA chains
  const bool lab_ok = (unsigned)lab <= 1u;             // labels other than 0/1 carry no residual block
  const float m = fmaf(cc.G, fabsf(x) + fabsf(y) + fabsf(z), cc.G0);
  float Z, al, ah;
  if (P == 4) {                                        // R = Ry: no y terms in X and Z
    Z = fmaf(cc.zc[0], x, fmaf(cc.zc[2], z, cc.zc[3]));
    al = fmaf(cc.al[0], x, fmaf(cc.al[2], z, cc.al[3]));
    ah = fmaf(cc.ah[0], x, fmaf(cc.ah[2], z, cc.ah[3]));
  } else {
    Z = fmaf(cc.zc[0], x, fmaf(cc.zc[1], y, fmaf(cc.zc[2], z, cc.zc[3])));
    al = fmaf(cc.al[0], x, fmaf(cc.al[1], y, fmaf(cc.al[2], z, cc.al[3])));
    ah = fmaf(cc.ah[0], x, fmaf(cc.ah[1], y, fmaf(cc.ah[2], z, cc.ah[3])));
  }
  const float bl = fmaf(cc.bl[0], x, fmaf(cc.bl[1], y, fmaf(cc.bl[2], z, cc.bl[3])));
  const float bh = fmaf(cc.bh[0], x, fmaf(cc.bh[1], y, fmaf(cc.bh[2], z, cc.bh[3])));
  // al > m, ah < -m, bl > m, bh < -m  <=>  lo4 > m ;   al < -m or ah > m or bl < -m or bh > m  <=>  lo4 < -m
  const float lo4 = fminf(fminf(al, -ah), fminf(bl, -bh));
  const bool front = Z > m;
  const bool inside = front && lo4 > m;                    // surely in the image
  const bool outside = (Z < -m) || (front && lo4 < -m);    // surely not
  const bool act = lab == 1 ? !inside : !outside;
  return lab_ok && (cc.enabled ? act : true);
}

// ------------------------------------------------------------------------------------------
// Box table.  The cloud of a sample is static over all of its (inits x evaluations) passes, so
// each group of 32 consecutive points gets an axis-aligned bounding box once per launch
// (frustum_boxes_kernel).  A linear form over a box ranges over  f(centre) +- sum |coef| half,
// so one lane decides a whole group against the five forms; only undecided groups are ever
// loaded point by point.  (frustum_prepare_batch sorts points by (label, Morton cell) so that
// groups are spatially compact and label-pure; unsorted clouds still work, they just cull less.)
//
// Global layout per sample: rounds x [8 fields][32] floats; round r holds 32 groups, one per lane, so a warp reads
// consecutive words -- groups r, r + R, r + 2R, ... of the cloud's R rounds (see frustum_boxes_kernel: every round is a
// uniform sample of the cloud, which balances the slices of a pass).  Fields: cx cy cz hx hy hz flags(bit0: has label 0,
// bit1: has label 1) pad.
// ------------------------------------------------------------------------------------------
constexpr int kBoxFields = 8;
constexpr int kRoundGroups = 32;                         // groups per round = one per lane
constexpr int kRoundPoints = kRoundGroups * 32;          // 1024 points
constexpr int kBoxRoundFloats = kBoxFields * kRoundGroups;
#ifndef DIB_RING
#define DIB_RING 128                          // pending-ring entries per warp and label (power of two)
#endif
#ifndef DIB_GPS
#define DIB_GPS 2                             // undecided groups fetched + classified per step
#endif
#ifndef DIB_SLICE_ROUNDS
#define DIB_SLICE_ROUNDS 4                    // rounds (of 1024 points) per slice: 20480 points = 20 rounds = 5 slices
#endif
#ifndef DIB_SMALL_SLICE_ROUNDS
#define DIB_SMALL_SLICE_ROUNDS 2              // rounds per slice of a small batch and of the late problems of a large one
#endif
#ifndef DIB_MAX_SLICES
#define DIB_MAX_SLICES 12
#endif
constexpr int kMaxSlices = DIB_MAX_SLICES;    // slices per pass held in shared memory (larger clouds get longer slices)

__host__ __device__ inline int box_rounds(int n) { return (n + kRoundPoints - 1) / kRoundPoints; }
// rounds per slice for a cloud of `rounds` rounds: the configured length, stretched for very large clouds so that
// the pass never has more than kMaxSlices slices.  Depends on the cloud size only (results must not depend on
// the batch or on who computes a slice).
__host__ __device__ inline int slice_len(int rounds, int want) {
  int len = want < 1 ? 1 : want;
  const int need = (rounds + kMaxSlices - 1) / kMaxSlices;
  return len < need ? need : len;
}

// Self-contained record of a point: the element of the packed per-launch copy and of the
// per-warp rings of maybe-active points.
template <typename CT> struct Entry;
template <> struct alignas(16) Entry<float> { float x, y, z; int lab; };
template <> struct alignas(16) Entry<double> { double x, y, z; long long lab; };

template <typename CT>
__global__ void __launch_bounds__(256) frustum_boxes_kernel(const CT* __restrict__ xyz,
                                                            const int8_t* __restrict__ label,
                                                            const int32_t* __restrict__ n_pts, int n_stride,
                                                            int rounds_max, float* __restrict__ table,
                                                            Entry<CT>* __restrict__ packed, int interleave) {
  const int s = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int gid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);     // destination: slot gid % 32 of round gid / 32
  if (gid >= rounds_max * kRoundGroups) return;
  const int n = n_pts ? n_pts[s] : n_stride;
  // Source group of this slot.  Consecutive groups of the (label, Morton)-sorted cloud are neighbours in space, and the
  // points with a non-zero residual sit along the frustum's border: in cloud order a fifth of the rounds would hold most
  // of a pass's exact-path work (measured: the heaviest 2-round slice has 4-6x the mean), and a pass that is cut into
  // slices is as slow as its heaviest slice.  So round r takes groups r, r + R, r + 2R, ... (R = the cloud's rounds):
  // every round, hence every slice, is a uniform sample of the cloud.
  int src = gid;
  if (interleave) {
    const int R = box_rounds(n);
    const int r = gid / kRoundGroups, q = gid % kRoundGroups;
    src = (r < R) ? q * R + r : rounds_max * kRoundGroups;              // rounds beyond the cloud's own stay empty
  }
  const int i_src = src * 32 + lane;
  const int i = gid * 32 + lane;
  double lo[3] = {1e300, 1e300, 1e300}, hi[3] = {-1e300, -1e300, -1e300};
  int lab = -1;
  Entry<CT> e;
  e.x = 0; e.y = 0; e.z = 0; e.lab = -1;
  if (i_src < n) {
    lab = label[(size_t)s * n_stride + i_src];
    if (lab == 0 || lab == 1) {
      e.x = xyz[((size_t)s * 3 + 0) * n_stride + i_src];
      e.y = xyz[((size_t)s * 3 + 1) * n_stride + i_src];
      e.z = xyz[((size_t)s * 3 + 2) * n_stride + i_src];
      e.lab = lab;
      lo[0] = hi[0] = (double)e.x; lo[1] = hi[1] = (double)e.y; lo[2] = hi[2] = (double)e.z;
    }
  }
  // packed copy: every slot of the sample's rounds x 32 x 32 grid is written (padding and ignored labels
  // as label -1), so the solver needs no bounds test
  packed[(size_t)s * rounds_max * kRoundPoints + i] = e;
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[c] = fmin(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], o));
      hi[c] = fmax(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], o));
    }
  const unsigned m0 = __ballot_sync(0xffffffffu, lab == 0), m1 = __ballot_sync(0xffffffffu, lab == 1);
  if (lane == 0) {
    const int r = gid / kRoundGroups, q = gid % kRoundGroups;
    float* rec = table + ((size_t)s * rounds_max + r) * kBoxRoundFloats + q;
    const int flags = (m0 ? 1 : 0) | (m1 ? 2 : 0);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float cf = 0.f, hf = 0.f;
      if (flags) {
        const double cd = 0.5 * (lo[c] + hi[c]);
        cf = (float)cd;
        // half extent measured from the ROUNDED centre, inflated so the fp32 box contains every point
        const double hd = fmax(hi[c] - (double)cf, (double)cf - lo[c]);
        hf = (float)(hd * 1.000001 + (fabs(cd) + hd) * 1.3e-7 + 1e-30);
      }
      rec[c * kRoundGroups] = cf;
      rec[(3 + c) * kRoundGroups] = hf;
    }
    rec[6 * kRoundGroups] = __int_as_float(flags);
    rec[7 * kRoundGroups] = 0.f;
  }
}

// ------------------------------------------------------------------------------------------
// Shared-memory layout.
// ------------------------------------------------------------------------------------------
struct LsSample {
  double x, value, gradient;
  int value_valid, gradient_valid;
};

template <int P>
struct LMState {
  static constexpr int NA = NAcc<P>::NA;
  double x[P], x_norm, cost, g[P], A[NA], grad_max;
  double scale[P], diag[P];
  double radius, dec;
  double step[P], delta[P], mcc;
  double lb[P], ub[P];
  double gd, dmax;
  LsSample lower, prev, cur;
  double xt[P];          // point of the pending evaluation
  int reuse_diag, step_ok, invalid, iteration, max_iter;
  int phase;             // 0 initial, 1 line-search sample, 2 candidate after failed line search, 3 cost at an infeasible start
  int ls_iter, evals, ls_steps, term;
};

constexpr int kBatch = 32;                // entries evaluated per exact-path batch (one per lane)
constexpr int kRing = DIB_RING;           // pending ring per label: < kBatch carried + at most DIB_GPS x 32 appended per step
static_assert(kBatch + 32 * DIB_GPS <= kRing, "ring too small");

// Scratch of the warp that EXECUTES a slice (its own or a CTA-mate's).
template <typename CT, int P>
struct WarpScratch {
  Entry<CT> ring[2][kRing];               // [label 0 | label 1] pending rings
  double accs[NAcc<P>::N][32];            // per-lane accumulators (column = lane: conflict-free)
};

// State of the problem a warp OWNS.  Helpers read pose/cls/cam/pk/box and write part[k]; everything else is
// touched by the owner only.
template <typename CT, int P>
struct ProbCtx {
  double part[kMaxSlices][NAcc<P>::N];    // slice sums of the open pass
  double tot[NAcc<P>::N];
  PoseConst pose;
  ClassConst cls;
  Cam cam;
  LMState<P> lm;
  const Entry<CT>* pk;                    // packed copy of the sample's cloud
  const float* box;                       // its box table
  int rounds, slice_rounds, nslices;      // of the OPEN pass (a young problem's pass is one slice, see open_pass)
  int len_full, nslices_full;             // the cloud's fixed slicing, used from pass number slice_after on
  int slice_after;                        // this problem's first sliced pass (0 for the late problems of a batch)
  int prob;
  int next_slice;                         // claim counter of the open pass (>= nslices: nothing left to claim)
  int done;                               // slices of the open pass that are finished
};

template <typename CT, int P>
struct Smem {
  WarpScratch<CT, P> scratch[Cfg<CT, P>::kWarps];
  ProbCtx<CT, P> ctx[Cfg<CT, P>::kWarps];
  unsigned open_mask;                     // bit w: warp w's open pass may still have unclaimed slices
  int n_active;                           // warps that own a problem or may still fetch one
};
static_assert(sizeof(Smem<float, 4>) * DIB_CTAS_PER_SM <= 227 * 1024, "4-DoF shared memory");
static_assert(sizeof(Smem<float, 6>) * DIB_CTAS_PER_SM <= 227 * 1024, "6-DoF shared memory");
static_assert(sizeof(Smem<double, 4>) * DIB_CTAS_PER_SM <= 227 * 1024, "4-DoF f64 shared memory");
static_assert(sizeof(Smem<double, 6>) * DIB_CTAS_PER_SM <= 227 * 1024, "6-DoF f64 shared memory");

// One box record as seven registers (cx cy cz hx hy hz flags).
struct BoxRec {
  float v[7];
};

__device__ __forceinline__ void box_load(const float* f, int slot, BoxRec& b) {
#pragma unroll
  for (int k = 0; k < 7; ++k) b.v[k] = __ldg(f + k * kRoundGroups + slot);
}

// Box test of one group by one lane.  0: every point of the group contributes exactly zero (skip); 1: undecided, the
// points must be classified one by one; 2: every point of the (label-pure) group is surely active -- a "should be
// outside" group that lies wholly inside the image or a "should be inside" group wholly outside it -- so its points go
// straight to the exact path without the per-point fp32 classification.
__device__ __forceinline__ int box_state(const BoxRec& b, const ClassConst& cc) {
  const int flags = __float_as_int(b.v[6]);
  if (flags == 0) return 0;                           // no point with a residual block
  if (!cc.enabled) return 1;
  const float cx = b.v[0], cy = b.v[1], cz = b.v[2], hx = b.v[3], hy = b.v[4], hz = b.v[5];
  const float m = 2.0f * fmaf(cc.G, (fabsf(cx) + hx) + (fabsf(cy) + hy) + (fabsf(cz) + hz), cc.G0);
  float lo[5], hi[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const float* c = cc.zc + 4 * k;                   // zc, al, ah, bl, bh are contiguous float[4]
    const float mid = fmaf(c[0], cx, fmaf(c[1], cy, fmaf(c[2], cz, c[3])));
    const float rad = fmaf(fabsf(c[0]), hx, fmaf(fabsf(c[1]), hy, fabsf(c[2]) * hz));
    lo[k] = mid - rad; hi[k] = mid + rad;
  }
  const bool front = lo[0] > m;
  const bool all_out = (hi[0] < -m) || (front && fminf(fminf(hi[1], -lo[2]), fminf(hi[3], -lo[4])) < -m);
  const bool all_in = front && fminf(fminf(lo[1], -hi[2]), fminf(lo[3], -hi[4])) > m;
  const bool skip = (!(flags & 1) || all_out) && (!(flags & 2) || all_in);
  if (skip) return 0;
  const bool sure = (flags == 1 && all_in) || (flags == 2 && all_out);
  return sure ? 2 : 1;
}

// ------------------------------------------------------------------------------------------
// One slice of a pass, executed by one warp (all 32 lanes call): rounds [r_begin, r_end) of the cloud.
// Box tests -> coalesced 16-byte loads of the undecided groups -> per-point fp32 culling -> ordered
// compaction into the executing warp's pending rings -> exact fp64 evaluation of 32 pending points at a time
// (one per lane, label-homogeneous) -> fixed-order reduction of the 32 lanes into part[0..N).
// The result depends only on (cloud, pose, r_begin, r_end): rings and accumulators start empty and are
// drained at the end of the slice, so any warp computes the same bits.
// ------------------------------------------------------------------------------------------
template <typename CT, int P>
__device__ __forceinline__ void eval_slice(WarpScratch<CT, P>& ws, const ProbCtx<CT, P>& pb, int r_begin, int r_end,
                                           double* part, int lane) {
  constexpr int N = NAcc<P>::N;
  const unsigned lt_mask = (1u << lane) - 1u;
  SmemAcc acc{&ws.accs[0][lane]};
#pragma unroll
  for (int j = 0; j < N; ++j) acc[j] = 0.0;
  const Cam& cam = pb.cam;
  const PoseConst& pc = pb.pose;
  const ClassConst& cc = pb.cls;
  const Entry<CT>* pk_s = pb.pk;
  const float* box_s = pb.box;
  Entry<CT>* ring0 = ws.ring[0];
  Entry<CT>* ring1 = ws.ring[1];
  int head0 = 0, pend0 = 0, head1 = 0, pend1 = 0;   // warp-uniform
  double prod = 1.0;                                  // per-lane product of (1 + s), renormalised
  int expo = 0;
  BoxRec box_cur, box_nxt;
#pragma unroll
  for (int k = 0; k < 7; ++k) { box_cur.v[k] = 0.f; box_nxt.v[k] = 0.f; }
  if (r_begin < r_end) box_load(box_s + (size_t)r_begin * kBoxRoundFloats, lane, box_nxt);

  // Rounds r_begin .. r_end-1 test one box per lane; the extra last round only drains what is left,
  // so each exact evaluator has ONE code instance.
#pragma unroll 1
  for (int r = r_begin; r <= r_end; ++r) {
    unsigned mask = 0, mask_sure = 0;       // undecided groups / groups whose points are all surely active
    int threshold = 1;
    if (r < r_end) {
      threshold = kBatch;
      box_cur = box_nxt;                              // loaded while the previous round was processed
      if (r + 1 < r_end) box_load(box_s + (size_t)(r + 1) * kBoxRoundFloats, lane, box_nxt);
      const int bs = box_state(box_cur, cc);
      mask = __ballot_sync(0xffffffffu, bs == 1);
      mask_sure = __ballot_sync(0xffffffffu, bs == 2);
    }
    // Undecided groups are taken DIB_GPS at a time.  Their loads are issued first, then the pending
    // exact-path batches are drained WHILE THE LOADS ARE IN FLIGHT, then the groups are classified
    // (independent instruction streams) and appended.  Ring bound: < kBatch carried + 32 x DIB_GPS new.
    // take the next DIB_GPS groups (surely-active ones first: a step made only of them skips the classification,
    // then the undecided ones) and issue their loads
    auto take_groups = [&](CT* lx, CT* ly, CT* lz, int* ll, bool& sure_only) -> bool {
      const bool any = (mask | mask_sure) != 0;
      sure_only = true;
      if (any) {
#pragma unroll
        for (int u = 0; u < DIB_GPS; ++u) {
          ll[u] = -1; lx[u] = 0; ly[u] = 0; lz[u] = 0;
          if (mask | mask_sure) {
            const bool from_sure = mask_sure != 0;
            const int b = __ffs(from_sure ? mask_sure : mask) - 1;
            if (from_sure) mask_sure &= mask_sure - 1; else mask &= mask - 1;
            sure_only = sure_only && from_sure;
            const Entry<CT> e = pk_s[(size_t)(r * kRoundGroups + b) * 32 + lane];      // this lane's point
            ll[u] = (int)e.lab; lx[u] = e.x; ly[u] = e.y; lz[u] = e.z;
          }
        }
      }
      return any;
    };
#pragma unroll 1
    do {
      // (issuing the NEXT step's loads before this step is classified -- a register software pipeline -- is not done:
      // the registers it needs cost more than the latency it hides)
      CT gx[DIB_GPS], gy[DIB_GPS], gz[DIB_GPS];
      int glab[DIB_GPS];
      bool all_sure = true;
      const bool have = take_groups(gx, gy, gz, glab, all_sure);
#pragma unroll 1
      while (pend0 >= threshold) {
        __syncwarp();
        const int take = pend0 < kBatch ? pend0 : kBatch;
        const Entry<CT> ea = ring0[(head0 + lane) & (kRing - 1)];
        Out0<P> oa;
        eval_outside<P>((double)ea.x, (double)ea.y, (double)ea.z, lane < take, cam, pc, oa);
        prod *= oa.s1;
        renorm_product(prod, expo);
        rank1<P, SmemAcc>(acc, oa.J, oa.w, oa.r);
        head0 = (head0 + take) & (kRing - 1);
        pend0 -= take;
      }
#pragma unroll 1
      while (pend1 >= threshold) {
        __syncwarp();
        const int take = pend1 < kBatch ? pend1 : kBatch;
        const Entry<CT> ea = ring1[(head1 + lane) & (kRing - 1)];
        Out1<P> oa;
        eval_inside<P>((double)ea.x, (double)ea.y, (double)ea.z, lane < take, cam, pc, oa);
        prod *= oa.s1;
        renorm_product(prod, expo);
        accumulate_inside<P, SmemAcc>(acc, oa);
        head1 = (head1 + take) & (kRing - 1);
        pend1 -= take;
      }
      if (have) {
        bool mb[DIB_GPS];
        if (all_sure) {                                  // warp-uniform: only padding / ignored labels drop out
#pragma unroll
          for (int u = 0; u < DIB_GPS; ++u) mb[u] = (unsigned)glab[u] <= 1u;
        } else {
          // The class constants (shared memory: every caller's ProbCtx lives there) are re-read here, six 128-bit loads
          // per step, instead of being held in ~20 registers from the round's box tests through the fp64 drains; the
          // volatile loads keep the compiler from hoisting them (DESIGN 4.4: 3-4 % faster on an H100).
          ClassConst ccr;
          {
            float4* d = reinterpret_cast<float4*>(&ccr);
            const uint32_t a = smem_u32(&cc);
#pragma unroll
            for (int q = 0; q < (int)(sizeof(ClassConst) / 16); ++q)
              asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                           : "=f"(d[q].x), "=f"(d[q].y), "=f"(d[q].z), "=f"(d[q].w) : "r"(a + 16 * q));
          }
#pragma unroll
          for (int u = 0; u < DIB_GPS; ++u) mb[u] = maybe_active<P>((float)gx[u], (float)gy[u], (float)gz[u], glab[u], ccr);
        }
#pragma unroll
        for (int u = 0; u < DIB_GPS; ++u) {
          const unsigned m1 = __ballot_sync(0xffffffffu, mb[u] && glab[u] == 1);
          const unsigned m0 = __ballot_sync(0xffffffffu, mb[u] && glab[u] == 0);
          if (mb[u]) {
            // one select + one store (the label picks ring, base and mask) instead of two predicated copies
            const bool l1 = glab[u] != 0;
            Entry<CT>* ring = l1 ? ring1 : ring0;
            const int at = (l1 ? head1 + pend1 : head0 + pend0) + __popc((l1 ? m1 : m0) & lt_mask);
            Entry<CT> e;
            e.x = gx[u]; e.y = gy[u]; e.z = gz[u]; e.lab = glab[u];
            ring[at & (kRing - 1)] = e;
          }
          pend0 += __popc(m0);
          pend1 += __popc(m1);
        }
      }
    } while (mask | mask_sure);
  }
  acc[0] = 0.5 * (log(prod) + (double)expo * 0.6931471805599453094);

  // Fixed-order reduction: lane j sums accumulator j over the 32 lanes, starting at column j (a fixed order per
  // accumulator; the rotation keeps the 32 reading lanes on 32 different banks).
  __syncwarp();
  if (lane < N) {
    double v = 0.0;
#pragma unroll 4
    for (int l = 0; l < 32; ++l) v += ws.accs[lane][(l + lane) & 31];   // rotated start: conflict-free, still a fixed order
    part[lane] = v;
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------
// Trust-region control flow (thread 0 only).
// ------------------------------------------------------------------------------------------
template <int P>
__device__ __forceinline__ void project_plus(const LMState<P>& st, const double* x, const double* d, double a, double* out) {
#pragma unroll
  for (int j = 0; j < P; ++j) {
    double v = fma(a, d[j], x[j]);
    v = fmax(v, st.lb[j]);
    v = fmin(v, st.ub[j]);
    out[j] = v;
  }
}

template <int P>
__device__ __forceinline__ double grad_max_norm(const LMState<P>& st, const double* x, const double* g) {
  double mx = 0.0;
#pragma unroll
  for (int j = 0; j < P; ++j) {
    double v = x[j] - g[j];
    v = fmax(v, st.lb[j]);
    v = fmin(v, st.ub[j]);
    mx = fmax(mx, fabs(x[j] - v));
  }
  return mx;
}

// Solve (As + diag(d2)) y = gs by Cholesky, As full symmetric P x P in registers.  One rsqrt per
// column and no divisions (the control code is latency-bound on one thread).  false if not SPD.
template <int P>
__device__ __forceinline__ bool chol_solve(const double (&As)[P][P], const double* d2, const double* gs, double* y) {
  double L[P][P], inv[P];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < P; ++j) {
    double s = As[j][j] + d2[j];
#pragma unroll
    for (int k = 0; k < j; ++k) s = fma(-L[j][k], L[j][k], s);
    if (!(s > 0.0)) ok = false;
    inv[j] = rsqrt(s);
    L[j][j] = s * inv[j];
#pragma unroll
    for (int i = j + 1; i < P; ++i) {
      double t = As[i][j];
#pragma unroll
      for (int k = 0; k < j; ++k) t = fma(-L[i][k], L[j][k], t);
      L[i][j] = t * inv[j];
    }
  }
  double z[P];
#pragma unroll
  for (int i = 0; i < P; ++i) {
    double t = gs[i];
#pragma unroll
    for (int k = 0; k < i; ++k) t = fma(-L[i][k], z[k], t);
    z[i] = t * inv[i];
  }
#pragma unroll
  for (int i = P - 1; i >= 0; --i) {
    double t = z[i];
#pragma unroll
    for (int k = i + 1; k < P; ++k) t = fma(-L[k][i], y[k], t);
    y[i] = t * inv[i];
  }
  return ok;
}

// ------------------------------------------------------------------------------------------
// Warp-collective line-search interpolation (every lane of the warp calls; the result is warp-uniform).
//
// Same algorithm as before -- the polynomial through the line-search samples from a full-pivot elimination of the
// Vandermonde-type system, its minimum over [xmin, xmax] from the real parts of ALL roots of the derivative, roots of
// cubics / quartics by Durand-Kerner -- but spread over the lanes: lane r holds row r of the system, a pivot search is
// a shuffle reduction with the serial scan's tie rule (first maximum in row-major order), row operations run in
// parallel, and every root of the derivative is iterated by its own lane (total-step Durand-Kerner: all roots are
// updated from the previous iterate).  The control step of a pass is on the critical path of its problem, and as
// straight-line single-lane code it was also ~50 KB of instructions that every problem dragged through the
// instruction cache once per pass; this version is ~4x shorter in both respects.
// ------------------------------------------------------------------------------------------
constexpr unsigned kFull = 0xffffffffu;

// Roots (real parts) of the monic polynomial c[0..deg], deg in {3, 4}, into roots[0..deg).
__device__ __forceinline__ void durand_kerner_warp(const double (&c)[5], int deg, double (&roots)[4], int lane) {
  // Fujiwara's bound on the root moduli: 2 max_k |c_k|^(1/k) (the last coefficient halved)
  double radius = 0.0;
#pragma unroll
  for (int i = 1; i <= 4; ++i) {
    if (i <= deg) {
      const double a = fabs(c[i]) * (i == deg ? 0.5 : 1.0);
      radius = fmax(radius, a > 0.0 ? exp(log(a) / (double)i) : 0.0);
    }
  }
  radius = 2.0 * radius + 1e-300;
  const int me = lane % deg;                      // every aligned group of 4 lanes holds all the roots
  double s, co;
  sincos(2.0 * 3.14159265358979323846 * me / deg + 0.4, &s, &co);   // start points on the circle of half that radius
  double zr = 0.5 * radius * co, zi = 0.5 * radius * s;
#pragma unroll 1
  for (int it = 0; it < 100; ++it) {
    double nr = 0.0, ni = 0.0;                    // p(z) by Horner
#pragma unroll
    for (int k = 0; k <= 4; ++k) {
      if (k <= deg) {
        const double tr = nr * zr - ni * zi + c[k];
        const double ti = nr * zi + ni * zr;
        nr = tr; ni = ti;
      }
    }
    double dr = 1.0, di = 0.0;                    // prod over the other roots of (z - z_j), j ascending
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j < deg) {
        const double zrj = __shfl_sync(kFull, zr, j), zij = __shfl_sync(kFull, zi, j);
        if (j != me) {
          const double er = zr - zrj, ei = zi - zij;
          const double tr = dr * er - di * ei, ti = dr * ei + di * er;
          dr = tr; di = ti;
        }
      }
    }
    double den = dr * dr + di * di;
    if (den == 0.0) { dr = 1e-300; di = 0.0; den = dr * dr; if (den == 0.0) den = 1e-300; }
    const double iden = 1.0 / den;
    const double qr = (nr * dr + ni * di) * iden, qi = (ni * dr - nr * di) * iden;
    zr -= qr; zi -= qi;
    double change = sqrt(qr * qr + qi * qi);
    change = fmax(change, __shfl_xor_sync(kFull, change, 1));
    change = fmax(change, __shfl_xor_sync(kFull, change, 2));
    if (change < 1e-14 * radius) break;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) roots[i] = __shfl_sync(kFull, zr, i);
}

// Step size minimising the polynomial that interpolates the line-search samples over [xmin, xmax] (cubic
// interpolation: values and gradients of lower / current / previous).
//
// The nc x nc system (nc <= 6) lives in the lanes: lane l holds M[l >> 3][l & 7] (rows 0..3) and, for l < 16,
// M[4 + (l >> 3)][l & 7] (rows 4, 5); column 6 is the right-hand side.  Every row operation of the serial full-pivot
// elimination is then one or two instructions for all elements at once, with the pivot row / column read by shuffles,
// and the loops over k are real loops (small code).  The arithmetic per element is that of the serial algorithm.
__device__ __forceinline__ double mat_fetch(double e0, double e1, int i, int j) {
  const int src = ((i & 3) << 3) | j;
  const double v0 = __shfl_sync(kFull, e0, src), v1 = __shfl_sync(kFull, e1, src);
  return i < 4 ? v0 : v1;
}

__device__ __noinline__ double interp_min_step_warp(const LsSample& lower, const LsSample& previous, const LsSample& current,
                                                    double xmin, double xmax, int lane) {
  if (!current.value_valid) return fmin(fmax(current.x * 0.5, xmin), xmax);
  const LsSample* smp[3] = {&lower, &current, &previous};
  const int ns = previous.value_valid ? 3 : 2;
  int nc = 0;
#pragma unroll 1
  for (int i = 0; i < ns; ++i) { nc += smp[i]->value_valid ? 1 : 0; nc += smp[i]->gradient_valid ? 1 : 0; }
  const int deg = nc - 1;
  const int j = lane & 7, i0 = lane >> 3, i1 = 4 + (lane >> 3);
  // element of row `r`, column j: value rows x^deg .. x^0, gradient rows deg x^(deg-1) .. 1 0, column 6 = rhs
  auto element = [&](int r) -> double {
    if (r >= nc || j == 7) return 0.0;
    int row = 0, kind = -1;
    double sx = 0.0, rhs = 0.0;
#pragma unroll 1
    for (int i = 0; i < ns; ++i) {
      if (smp[i]->value_valid) { if (row == r) { sx = smp[i]->x; rhs = smp[i]->value; kind = 0; } ++row; }
      if (smp[i]->gradient_valid) { if (row == r) { sx = smp[i]->x; rhs = smp[i]->gradient; kind = 1; } ++row; }
    }
    if (j == 6) return rhs;
    const int e = (kind == 0) ? deg - j : deg - j - 1;      // exponent of x in this entry
    if (e < 0) return 0.0;
    double pw = 1.0;                                       // x^e by repeated multiplication
#pragma unroll 1
    for (int q = 0; q < e; ++q) pw = pw * sx;
    return (kind == 0) ? pw : (double)(e + 1) * pw;
  };
  double e0 = element(i0), e1 = (lane < 16) ? element(i1) : 0.0;

  // full-pivot elimination (column permutation packed in one register, 4 bits per entry)
  unsigned perm = 0x543210u;
#pragma unroll 1
  for (int k = 0; k < nc; ++k) {
    // pivot: first maximum of |M[i][j]| over i, j in [k, nc) in row-major order
    double val = -1.0;
    int idx = 0x7fffffff;
    if (j >= k && j < nc) {
      if (i0 >= k && i0 < nc) { val = fabs(e0); idx = i0 * 8 + j; if (!(val > -1.0)) { val = -1.0; } }
      if (lane < 16 && i1 >= k && i1 < nc) {
        const double v1 = fabs(e1);
        if (v1 > val) { val = v1; idx = i1 * 8 + j; }
        else if (idx == 0x7fffffff) idx = i1 * 8 + j;
      }
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double ov = __shfl_xor_sync(kFull, val, o);
      const int oi = __shfl_xor_sync(kFull, idx, o);
      if (ov > val || (ov == val && oi < idx)) { val = ov; idx = oi; }
    }
    if (val < 0.0) idx = k * 8 + k;                 // nothing comparable (NaNs): the serial scan keeps (k, k)
    if (val == 0.0) {                               // singular: remaining right-hand sides are zeroed, elimination stops
      if (j == 6) { if (i0 >= k && i0 < nc) e0 = 0.0; if (lane < 16 && i1 >= k && i1 < nc) e1 = 0.0; }
      break;
    }
    const int pr = idx >> 3, pcv = idx & 7;
    if (pr != k) {                                  // row swap (all columns and the rhs)
      const double ak0 = mat_fetch(e0, e1, k, j), ap0 = mat_fetch(e0, e1, pr, j);
      if (i0 == k) e0 = ap0; else if (i0 == pr) e0 = ak0;
      if (i1 == k) e1 = ap0; else if (i1 == pr) e1 = ak0;
    }
    if (pcv != k) {                                 // column swap (all rows)
      const int jo = (j == k) ? pcv : ((j == pcv) ? k : j);
      const double n0 = __shfl_sync(kFull, e0, (i0 << 3) | jo), n1 = __shfl_sync(kFull, e1, (i0 << 3) | jo);
      e0 = n0; e1 = n1;
      const unsigned pa = (perm >> (4 * pcv)) & 15u, pb = (perm >> (4 * k)) & 15u;
      perm = (perm & ~((15u << (4 * pcv)) | (15u << (4 * k)))) | (pb << (4 * pcv)) | (pa << (4 * k));
    }
    // M[i][j] -= (M[i][k] / M[k][k]) M[k][j] for i > k, j >= k (rhs included)
    const double pkk = mat_fetch(e0, e1, k, k);
    const double pkj = mat_fetch(e0, e1, k, j);
    const double a0 = __shfl_sync(kFull, e0, (i0 << 3) | k), a1 = __shfl_sync(kFull, e1, (i0 << 3) | k);
    if (j >= k && (j < nc || j == 6)) {
      if (i0 > k && i0 < nc) { const double f = a0 / pkk; e0 -= f * pkj; }
      if (lane < 16 && i1 > k && i1 < nc) { const double f = a1 / pkk; e1 -= f * pkj; }
    }
  }
  // back substitution: z[k] kept by lane k
  double zmine = 0.0;
#pragma unroll 1
  for (int k = nc - 1; k >= 0; --k) {
    const double mkk = mat_fetch(e0, e1, k, k);
    double sacc = mat_fetch(e0, e1, k, 6);
#pragma unroll 1
    for (int jj = k + 1; jj < nc; ++jj) sacc -= mat_fetch(e0, e1, k, jj) * __shfl_sync(kFull, zmine, jj);
    const double zk = (mkk == 0.0) ? 0.0 : sacc / mkk;
    if (lane == k) zmine = zk;
  }
  // poly[perm[k]] = z[k]; coefficient c of the polynomial kept by lane c (highest power first)
  double pmine = 0.0;
#pragma unroll 1
  for (int k = 0; k < nc; ++k) {
    const double zk = __shfl_sync(kFull, zmine, k);
    if (lane == (int)((perm >> (4 * k)) & 15u)) pmine = zk;
  }
  auto poly_at = [&](double x) -> double {
    double v = 0.0;
#pragma unroll 1
    for (int i = 0; i < nc; ++i) v = v * x + __shfl_sync(kFull, pmine, i);
    return v;
  };
  double best_x = (xmin + xmax) / 2.0;
  double best_v = poly_at(best_x);
  const double vmin = poly_at(xmin);
  if (vmin < best_v) { best_v = vmin; best_x = xmin; }
  const double vmax = poly_at(xmax);
  if (vmax < best_v) { best_v = vmax; best_x = xmax; }
  if (nc <= 2) return best_x;
  // derivative (deg coefficients, lane jj holds coefficient jj), leading zeros stripped
  const double dmine = (lane < deg) ? (double)(deg - lane) * pmine : 0.0;
  const unsigned zmask = __ballot_sync(kFull, lane < deg && dmine == 0.0);
  int lead = __ffs(~zmask) - 1;
  if (lead > deg) lead = deg;
  const double qmine = __shfl_sync(kFull, dmine, (lane + lead) & 31);     // q[i] = der[lead + i]
  const int rdeg = deg - lead - 1;
  double roots[4] = {0.0, 0.0, 0.0, 0.0};
  int nr = 0;
  if (rdeg == 1) {
    roots[0] = -__shfl_sync(kFull, qmine, 1) / __shfl_sync(kFull, qmine, 0);
    nr = 1;
  } else if (rdeg == 2) {
    const double a = __shfl_sync(kFull, qmine, 0), b = __shfl_sync(kFull, qmine, 1), c = __shfl_sync(kFull, qmine, 2);
    const double D = b * b - 4 * a * c;
    const double sD = sqrt(fabs(D));
    if (D >= 0) {
      if (b >= 0) { roots[0] = (-b - sD) / (2.0 * a); roots[1] = (2.0 * c) / (-b - sD); }
      else { roots[0] = (2.0 * c) / (-b + sD); roots[1] = (-b + sD) / (2.0 * a); }
    } else { roots[0] = -b / (2.0 * a); roots[1] = roots[0]; }
    nr = 2;
  } else if (rdeg >= 3) {
    const double ip0 = 1.0 / __shfl_sync(kFull, qmine, 0);
    double c[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) c[i] = __shfl_sync(kFull, qmine, i) * ip0;
    durand_kerner_warp(c, rdeg, roots, lane);
    nr = rdeg;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (i < nr && !(roots[i] < xmin || roots[i] > xmax)) {
      const double v = poly_at(roots[i]);
      if (v < best_v) { best_v = v; best_x = roots[i]; }
    }
  }
  return best_x;
}

enum { LM_DONE = 0, LM_EVAL = 1, LM_INTERP = 2 };

// Starts the next trust-region iteration(s) until an evaluation is needed or the solve ends.
template <int P>
__device__ __noinline__ int lm_next_step(LMState<P>& st) {
  for (;;) {
    if (st.iteration >= st.max_iter) { st.term = 3; return LM_DONE; }
    if (st.step_ok && st.grad_max <= 1e-10) { st.term = 0; return LM_DONE; }
    if (st.radius <= 1e-32) { st.term = 4; return LM_DONE; }
    ++st.iteration;
    st.step_ok = 0;

    double As[P][P], gs[P], d2[P], y[P], sc[P];
#pragma unroll
    for (int j = 0; j < P; ++j) { sc[j] = st.scale[j]; gs[j] = st.g[j] * sc[j]; }
    {
      int idx = 0;
#pragma unroll
      for (int j = 0; j < P; ++j)
#pragma unroll
        for (int k = j; k < P; ++k) {
          const double v = st.A[idx++] * sc[j] * sc[k];
          As[j][k] = v; As[k][j] = v;
        }
    }
    if (!st.reuse_diag) {
#pragma unroll
      for (int j = 0; j < P; ++j) st.diag[j] = fmin(fmax(As[j][j], 1e-6), 1e32);
    }
    st.reuse_diag = 1;
    {
      const double inv_radius = 1.0 / st.radius;      // D^2 = diag / radius (LM damping)
#pragma unroll
      for (int j = 0; j < P; ++j) d2[j] = st.diag[j] * inv_radius;
    }
    bool ok = chol_solve<P>(As, d2, gs, y);
    double mcc = 0.0;
    if (ok) {
      // model cost change = -step^T gs - 1/2 step^T As step, step = -y
      double quad = 0.0, lin = 0.0;
#pragma unroll
      for (int j = 0; j < P; ++j) {
        st.step[j] = -y[j];
        if (!isfinite(y[j])) ok = false;
      }
#pragma unroll
      for (int j = 0; j < P; ++j) {
        lin = fma(-y[j], gs[j], lin);
        double rowsum = 0.0;
#pragma unroll
        for (int k = 0; k < P; ++k) rowsum = fma(As[j][k], -y[k], rowsum);
        quad = fma(-y[j], rowsum, quad);
      }
      mcc = -lin - 0.5 * quad;
    }
    if (!ok || !(mcc > 0.0)) {
      if (++st.invalid >= 5) { st.term = 5; return LM_DONE; }
      st.radius = st.radius / st.dec;      // LevenbergMarquardtStrategy::StepIsInvalid() == StepRejected(0)
      st.dec *= 2.0;
      st.reuse_diag = 1;
      continue;
    }
    st.invalid = 0;
    st.mcc = mcc;
    double gd = 0.0, dmax = 0.0;
#pragma unroll
    for (int j = 0; j < P; ++j) {
      st.delta[j] = st.step[j] * st.scale[j];
      gd += st.g[j] * st.delta[j];
      dmax = fmax(dmax, fabs(st.delta[j]));
    }
    st.gd = gd; st.dmax = dmax;
    st.lower.x = 0.0; st.lower.value = st.cost; st.lower.gradient = gd; st.lower.value_valid = 1; st.lower.gradient_valid = 1;
    st.prev.value_valid = 0; st.prev.gradient_valid = 0; st.prev.x = 0; st.prev.value = 0; st.prev.gradient = 0;
    st.cur.x = 1.0;
    st.ls_iter = 0;
    project_plus<P>(st, st.x, st.delta, 1.0, st.xt);
    st.phase = 1;
    return LM_EVAL;
  }
}

template <int P>
__device__ __noinline__ int lm_after_candidate(LMState<P>& st, const double* tot) {
  constexpr int NA = NAcc<P>::NA;
  const double ccost = tot[0];
  double sn = 0.0;
#pragma unroll
  for (int j = 0; j < P; ++j) sn += (st.x[j] - st.xt[j]) * (st.x[j] - st.xt[j]);
  if (sqrt(sn) <= 1e-8 * (st.x_norm + 1e-8)) { st.term = 1; return LM_DONE; }
  if (fabs(st.cost - ccost) <= 1e-6 * st.cost) { st.term = 2; return LM_DONE; }
  const double rho = (st.cost - ccost) / st.mcc;
  if (rho > 1e-3) {
    double xn = 0.0;
#pragma unroll
    for (int j = 0; j < P; ++j) { st.x[j] = st.xt[j]; xn += st.x[j] * st.x[j]; st.g[j] = tot[1 + j]; }
    st.x_norm = sqrt(xn);
    st.cost = ccost;
#pragma unroll
    for (int j = 0; j < NA; ++j) st.A[j] = tot[1 + P + j];
    st.grad_max = grad_max_norm<P>(st, st.x, st.g);
    const double t = 2.0 * rho - 1.0;
    st.radius = st.radius / fmax(1.0 / 3.0, 1.0 - t * t * t);
    st.radius = fmin(1e16, st.radius);
    st.dec = 2.0;
    st.reuse_diag = 0;
    st.step_ok = 1;
  } else {
    st.radius = st.radius / st.dec;
    st.dec *= 2.0;
    st.reuse_diag = 1;
  }
  return lm_next_step<P>(st);
}

template <int P>
__device__ __noinline__ int lm_consume_step(LMState<P>& st, double a, bool fail);

// Consumes the evaluation at st.xt (totals in tot).  Returns LM_EVAL with a new st.xt, LM_DONE, or LM_INTERP when the
// line search needs an interpolated step size (interp_min_step_warp, then lm_consume_step).
template <int P>
__device__ __noinline__ int lm_consume(LMState<P>& st, const double* tot) {
  constexpr int NA = NAcc<P>::NA;
  if (st.phase == 3) {                     // infeasible start: Problem::Evaluate at the untouched init, no solve
    st.cost = tot[0];
    return LM_DONE;
  }
  ++st.evals;
  if (st.phase == 0) {
    st.cost = tot[0];
    #pragma unroll 1
    for (int j = 0; j < P; ++j) st.g[j] = tot[1 + j];
    #pragma unroll 1
    for (int j = 0; j < NA; ++j) st.A[j] = tot[1 + P + j];
    #pragma unroll 1
    for (int j = 0; j < P; ++j) st.scale[j] = 1.0 / (1.0 + sqrt(st.A[tri(P, j, j)]));
    st.grad_max = grad_max_norm<P>(st, st.x, st.g);
    st.step_ok = 1;
    return lm_next_step<P>(st);
  }
  if (st.phase == 1) {
    LsSample& cur = st.cur;
    cur.value = tot[0];
    cur.value_valid = isfinite(cur.value) ? 1 : 0;
    double gr = 0.0;
    #pragma unroll 1
    for (int j = 0; j < P; ++j) gr += st.delta[j] * tot[1 + j];
    cur.gradient = gr;
    cur.gradient_valid = (cur.value_valid && isfinite(gr)) ? 1 : 0;
    const bool armijo_ok = cur.value_valid && !(cur.value > st.cost + 1e-4 * st.gd * cur.x);
    if (armijo_ok) {
      #pragma unroll 1
      for (int j = 0; j < P; ++j) st.delta[j] *= cur.x;
      return lm_after_candidate<P>(st, tot);      // candidate == this sample, bit for bit
    }
    ++st.ls_iter;
    ++st.ls_steps;
    if (st.ls_iter < 20) return LM_INTERP;    // the warp computes the interpolated step, then lm_consume_step() goes on
    return lm_consume_step<P>(st, 0.0, true);
  }
  return lm_after_candidate<P>(st, tot);
}

// Second half of a failed Armijo test: `a` is the step size from the warp-collective interpolation (or `fail` is set
// because the line search ran out of iterations).
template <int P>
__device__ __noinline__ int lm_consume_step(LMState<P>& st, double a, bool fail) {
  {
    LsSample& cur = st.cur;
    if (!fail && a * st.dmax < 1e-9) fail = true;
    if (fail) {
      // line search failed: the full step is the candidate (delta untouched)
      project_plus<P>(st, st.x, st.delta, 1.0, st.xt);
      st.phase = 2;
      return LM_EVAL;
    }
    st.prev = cur;
    cur.x = a;
    {
      double sd[P];
      #pragma unroll 1
      for (int j = 0; j < P; ++j) sd[j] = a * st.delta[j];
      project_plus<P>(st, st.x, sd, 1.0, st.xt);
    }
    return LM_EVAL;
  }
}

// Sets st.xt and returns LM_EVAL (an infeasible start asks for ONE cost-only pass at the init, phase 3).
template <int P>
__device__ __noinline__ int lm_begin(LMState<P>& st, const double* init4, const double* lb3, const double* ub3, int max_iter) {
  constexpr int toff = P - 3;
  #pragma unroll 1
  for (int j = 0; j < P; ++j) { st.lb[j] = -DBL_MAX; st.ub[j] = DBL_MAX; st.x[j] = 0.0; }
  #pragma unroll 1
  for (int k = 0; k < 3; ++k) { st.lb[toff + k] = lb3[k]; st.ub[toff + k] = ub3[k]; st.x[toff + k] = init4[1 + k]; }
  st.x[P == 4 ? 0 : 1] = init4[0];        // registration.cpp:34-50
  st.max_iter = max_iter;
  st.iteration = 0; st.evals = 0; st.ls_steps = 0; st.term = -1; st.invalid = 0;
  st.radius = 1e4; st.dec = 2.0; st.reuse_diag = 0; st.step_ok = 1; st.phase = 0;
  st.cost = 0.0; st.grad_max = 0.0; st.mcc = 0.0; st.cur.x = 1.0;
  #pragma unroll 1
  for (int j = 0; j < P; ++j) st.g[j] = 0.0;
  #pragma unroll 1
  for (int j = 0; j < P; ++j)
    if (st.x[j] < st.lb[j] || st.x[j] > st.ub[j]) { st.term = 6; st.phase = 3; }
  double xn = 0.0;
  #pragma unroll 1
  for (int j = 0; j < P; ++j) { st.xt[j] = st.x[j]; xn += st.x[j] * st.x[j]; }
  st.x_norm = sqrt(xn);
  return LM_EVAL;                          // always: an infeasible start still gets its cost evaluated (phase 3)
}

__device__ void make_cam(const double* K9, double H, double W, Cam* cam) {
  cam->fx = K9[0]; cam->fy = K9[4]; cam->cx = K9[2]; cam->cy = K9[5];   // registration.cpp:79-82
  cam->W1 = W - 1.0; cam->H1 = H - 1.0;                                 // registration.cpp:21-22
  cam->hW = cam->W1 * 0.5; cam->hH = cam->H1 * 0.5;
}

struct SolveArgs {
  const void* xyz;
  const int8_t* label;
  const int32_t* n_pts;
  int n_stride;
  const double* K9;
  const double* init;
  double lb[3], ub[3];
  double H, W;
  int max_iter, S, I;
  double* params_all;   // [S*I*6]
  double* cost_all;     // [S*I]
  int32_t* stats_all;   // [S*I*4]
  unsigned int* queue;  // problem counter (problems beyond the statically assigned first wave)
  const float* boxes;   // [S][rounds_max][8][32] box table
  const void* packed;   // [S][rounds_max * 1024] Entry<CT>
  int rounds_max;
  const int32_t* perm;  // [S][I] inits of each sample, longest-predicted first
  int chunk;            // samples per scheduling chunk
  int slice_rounds;     // rounds per slice (before the kMaxSlices stretch)
  int slice_after;      // passes of a problem that run as ONE slice before the fixed slicing starts
  int late_from;        // queue positions >= late_from are LATE problems: sliced from their first pass, in
  int late_slice_rounds; // slices of late_slice_rounds rounds (they run while the batch drains: help is there from the start)
  double* trace;        // optional [S*I][trace_cap][kTraceRec] per-evaluation records, or NULL
  int trace_cap;
};

constexpr int kCtaEndSlots = 1024;   // per-CTA exit times kept after the workspace header (benchmark timeline)
constexpr size_t kHeaderBytes = 256 + kCtaEndSlots * 8;
constexpr int kTraceRec = 16;   // doubles per trace record, see include/deepi2p_b200.h (frustum_solve_traced_*)

// Scheduling order.  Solve length correlates with how far an init's heading is from the centre of its
// sample's inits (rank correlation ~0.6 with the number of evaluations), so each sample's inits are
// ranked by that distance, longest-predicted first, and the queue walks chunks of samples rank-major:
// the expensive solves start early, while concurrently running problems still share an L2-sized set of clouds.
// perm [S][I]: perm[s][r] = init index of rank r.  Results do not depend on the order.
__global__ void frustum_order_kernel(const double* __restrict__ init, int I, int32_t* __restrict__ perm) {
  extern __shared__ double key[];
  const int s = blockIdx.x;
  const double* in = init + (size_t)s * I * 4;
  double mean = 0.0;
  for (int i = 0; i < I; ++i) mean += in[(size_t)i * 4];       // every thread: same fixed-order sum
  mean /= (double)I;
  for (int i = threadIdx.x; i < I; i += blockDim.x) key[i] = fabs(in[(size_t)i * 4] - mean);
  __syncthreads();
  for (int i = threadIdx.x; i < I; i += blockDim.x) {
    const double k = key[i];
    int rank = 0;
    for (int j = 0; j < I; ++j) {
      const double kj = key[j];
      rank += (kj > k || (kj == k && j < i)) ? 1 : 0;       // NaN keys compare false: ties by index
    }
    perm[(size_t)s * I + rank] = i;
  }
}

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ int ld_volatile(const int* p) { return *reinterpret_cast<const volatile int*>(p); }
__device__ __forceinline__ unsigned ld_volatile(const unsigned* p) { return *reinterpret_cast<const volatile unsigned*>(p); }
__device__ __forceinline__ void st_volatile(int* p, int v) { *reinterpret_cast<volatile int*>(p) = v; }

// Lane 0 of the owner: publish the pass whose pose / classification constants were just written.
// A pass is cut into slices only from the problem's slice_after-th pass on: short solves (most of them) never pay the
// per-slice overhead (rings drained and accumulators reduced at every slice end), while the long solves that make up
// the end-of-kernel tail can be helped.  The switch depends on the problem's own pass count only, so results stay
// independent of the batch, of the schedule and of who helps.
template <typename CT, int P>
__device__ __forceinline__ void open_pass(Smem<CT, P>& sm, ProbCtx<CT, P>& me, int warp) {
  const bool sliced = me.lm.evals >= me.slice_after;
  // Close the counter before the slice layout changes: after a pass next_slice equals the OLD slice count, which is
  // below the new one when a problem goes from one-piece to sliced passes -- a helper polling in that window would
  // claim a slice of a pass that is not open yet (and be counted twice).
  st_volatile(&me.next_slice, 0x3fffffff);
  __threadfence_block();
  me.nslices = sliced ? me.nslices_full : 1;
  me.slice_rounds = sliced ? me.len_full : (me.rounds > 0 ? me.rounds : 1);
  st_volatile(&me.done, 0);
  __threadfence_block();                       // pose, cls, layout, done before the pass becomes claimable
  // only a pass with more than one slice is advertised: a one-piece pass is its owner's alone (a "helper" would just
  // take the whole pass away while the owner waits)
  if (me.nslices > 1) atomicOr(&sm.open_mask, 1u << warp);   // bit first: whoever claims the last slice clears it again
  st_volatile(&me.next_slice, 0);
}

template <typename CT, int P>
__device__ __forceinline__ void trace_record(const SolveArgs& a, const ProbCtx<CT, P>& me, int rec_idx, bool after) {
  if (a.trace == nullptr || rec_idx >= a.trace_cap) return;
  double* t = a.trace + ((size_t)me.prob * a.trace_cap + rec_idx) * kTraceRec;
  const LMState<P>& st = me.lm;
  if (!after) {
    for (int j = 0; j < 6; ++j) t[j] = j < P ? st.xt[j] : 0.0;
    t[6] = me.tot[0];
    t[7] = st.cost;
    t[8] = st.radius;
    t[9] = (double)st.iteration;
    t[10] = (double)st.phase;
    t[13] = st.phase == 1 ? st.cur.x : 1.0;
    t[14] = st.mcc;
    t[15] = 1.0;                               // record valid
  } else {
    bool moved = true;                         // the evaluated point became the iterate <=> x == x_t now
    for (int j = 0; j < P; ++j) moved = moved && (st.x[j] == t[j]);
    t[11] = moved ? 1.0 : 0.0;
    t[12] = (double)st.term;                   // -1 while running
  }
}

enum { ST_FETCH = 0, ST_RUN = 1, ST_IDLE = 2 };

template <typename CT, int P>
__global__ void __launch_bounds__(Cfg<CT, P>::kWarps * 32, DIB_CTAS_PER_SM) frustum_solve_kernel(SolveArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem<CT, P>& sm = *reinterpret_cast<Smem<CT, P>*>(smem_raw);
  constexpr int kW = Cfg<CT, P>::kWarps;
  constexpr int N = NAcc<P>::N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  ProbCtx<CT, P>& me = sm.ctx[warp];
  WarpScratch<CT, P>& ws = sm.scratch[warp];
  if (lane == 0) { me.next_slice = 0x3fffffff; me.nslices = 0; me.done = 0; me.prob = -1; }
  if (threadIdx.x == 0) { sm.open_mask = 0u; sm.n_active = kW; }
  // Launch timeline for the benchmark (three 64-bit words after the queue counter, zeroed / primed by the host):
  // kernel start, the moment the queue ran dry, the last CTA's exit -- all in globaltimer nanoseconds.
  unsigned long long* tl = reinterpret_cast<unsigned long long*>(a.queue) + 1;
  unsigned long long* cta_end = reinterpret_cast<unsigned long long*>(a.queue) + 32;   // [kCtaEndSlots], after the 256-byte header
  if (threadIdx.x == 0) atomicMin(tl + 0, global_ns());
  __syncthreads();                               // the only CTA-wide barrier of the kernel
  const int total = a.S * a.I;
  int state = ST_FETCH;                          // warp-uniform
  bool first = true;
  int n_rec = 0;                                 // trace records written for the current problem (lane 0)
#ifdef DIB_PASS_TIMING
  unsigned long long t_open = global_ns();
#endif

  for (;;) {
    if (state == ST_FETCH) {
      // First wave: problem ranks are dealt statically, rank-major over the CTAs, so that a batch smaller than
      // the grid's warp count leaves every CTA with idle warps that help; later problems come from the queue.
      int q = 0;
      if (first) { q = warp * (int)gridDim.x + (int)blockIdx.x; first = false; }
      else {
        if (lane == 0) q = (int)gridDim.x * kW + (int)atomicAdd(a.queue, 1u);
        q = __shfl_sync(0xffffffffu, q, 0);
      }
      if (q >= total) {
        state = ST_IDLE;
        if (lane == 0) { atomicSub(&sm.n_active, 1); atomicMin(tl + 1, global_ns()); }
        continue;
      }
      const int per_chunk = a.chunk * a.I;
      const int c = q / per_chunk, within = q - c * per_chunk;
      const int s0 = c * a.chunk;
      const int gc = min(a.chunk, a.S - s0);             // samples in this chunk
      const int rk = within / gc, s = s0 + (within - rk * gc);
      const int prob = s * a.I + a.perm[(size_t)s * a.I + rk];
      int rc = LM_DONE;
      if (lane == 0) {
        const int n = a.n_pts ? a.n_pts[s] : a.n_stride;
        const int rounds = box_rounds(n);
        const bool late = q >= a.late_from;
        const int len = slice_len(rounds, late ? a.late_slice_rounds : a.slice_rounds);
        me.slice_after = late ? 0 : a.slice_after;
        me.prob = prob;
        me.pk = reinterpret_cast<const Entry<CT>*>(a.packed) + (size_t)s * a.rounds_max * kRoundPoints;
        me.box = a.boxes + (size_t)s * a.rounds_max * kBoxRoundFloats;
        me.rounds = rounds;
        me.len_full = len;
        me.nslices_full = rounds > 0 ? (rounds + len - 1) / len : 1;    // an empty cloud still has one (empty) slice
        make_cam(a.K9 + (size_t)s * 9, a.H, a.W, &me.cam);
        rc = lm_begin<P>(me.lm, a.init + (size_t)prob * 4, a.lb, a.ub, a.max_iter);
        n_rec = 0;
        if (rc == LM_EVAL) make_pose<P>(me.lm.xt, &me.pose);
      }
      __syncwarp();                                     // lane 0's problem set-up is visible to the whole warp
      rc = __shfl_sync(0xffffffffu, rc, 0);
      if (rc == LM_EVAL) {
        make_class(me.pose, me.cam, &me.cls, lane);
        __syncwarp();
        if (lane == 0) open_pass<CT, P>(sm, me, warp);
        __syncwarp();
#ifdef DIB_PASS_TIMING
        t_open = global_ns();
#endif
      }
      state = (rc == LM_EVAL) ? ST_RUN : ST_FETCH;        // lm_begin always asks for an evaluation today
      continue;
    }

    // ---- pick a slice: my own finished pass first, then a slice of mine, else any open pass of a CTA-mate ----
    // (taking the open slices of OLD problems before a warp's own work -- "oldest first" -- measured no gain, 79.1 vs
    // 78.5 ms: the end-of-kernel tail is in-flight work draining at falling occupancy, not old problems running slowly)
    int owner = -1, k = 0, r_begin = 0, r_end = 0;
    // lane 0 tries to claim a slice of the lowest-numbered warp in `m`; returns the warp (or -1) and the slice in kk
    auto try_claim = [&](unsigned m, int& kk) -> int {
      int o = -1;
      if (lane == 0 && m) {
        const int cand = __ffs(m) - 1;
        ProbCtx<CT, P>& oc = sm.ctx[cand];
        if (ld_volatile(&oc.next_slice) < ld_volatile(&oc.nslices)) {
          const int got = atomicAdd(&oc.next_slice, 1);
          __threadfence_block();
          const int ns = ld_volatile(&oc.nslices);        // re-read after the claim: the pass cannot change under a valid claim
          if (got < ns) {
            o = cand; kk = got;
            if (got == ns - 1) atomicAnd(&sm.open_mask, ~(1u << cand));
          }
        }
      }
      __syncwarp();
      o = __shfl_sync(0xffffffffu, o, 0);
      kk = __shfl_sync(0xffffffffu, kk, 0);
      return o;
    };
    // my own finished pass comes first: only I can take its control step, and it is the serial part of my problem
    int complete = 0;
    if (state == ST_RUN) {
      if (lane == 0) {
        const int ns = me.nslices;
        complete = (ld_volatile(&me.next_slice) >= ns && ld_volatile(&me.done) == ns) ? 1 : 0;
      }
      complete = __shfl_sync(0xffffffffu, complete, 0);
    }
    if (owner < 0 && state == ST_RUN) {
      int mine = -1;
      if (lane == 0 && !complete) {
        const int ns = me.nslices;
        if (ld_volatile(&me.next_slice) < ns) {
          const int kk = atomicAdd(&me.next_slice, 1);
          if (kk < ns) {
            mine = kk;
            if (kk == ns - 1) atomicAnd(&sm.open_mask, ~(1u << warp));
          }
        }
      }
      mine = __shfl_sync(0xffffffffu, mine, 0);
      if (mine >= 0) {
        owner = warp; k = mine;
      } else if (complete) {
        // every slice of my pass is in: add the slice sums in slice order, then lane 0 takes the control step
        __threadfence_block();
        const int ns = me.nslices;
        if (lane < N) {
          double v = me.part[0][lane];
          for (int j = 1; j < ns; ++j) v += me.part[j][lane];
          me.tot[lane] = v;
        }
        __syncwarp();
        int rc = LM_DONE;
#ifdef DIB_PASS_TIMING
        const unsigned long long t_complete = global_ns();
#endif
        if (lane == 0) {
          trace_record<CT, P>(a, me, n_rec, false);
          rc = lm_consume<P>(me.lm, me.tot);
        }
        __syncwarp();
        rc = __shfl_sync(0xffffffffu, rc, 0);
        if (rc == LM_INTERP) {                      // warp-collective: interpolated line-search step size
          const LMState<P>& st = me.lm;
          const double step = interp_min_step_warp(st.lower, st.prev, st.cur, 1e-3 * st.cur.x, 0.6 * st.cur.x, lane);
          __syncwarp();                             // every lane is done reading the samples before lane 0 rewrites them
          if (lane == 0) rc = lm_consume_step<P>(me.lm, step, false);
        }
        if (lane == 0) {
          trace_record<CT, P>(a, me, n_rec, true);
          ++n_rec;
          if (rc == LM_EVAL) {
            make_pose<P>(me.lm.xt, &me.pose);
          } else {
            const LMState<P>& st = me.lm;
            double* po = a.params_all + (size_t)me.prob * 6;
            for (int j = 0; j < 6; ++j) po[j] = (j < P) ? st.x[j] : 0.0;
            a.cost_all[me.prob] = st.cost;
            int32_t* so = a.stats_all + (size_t)me.prob * 4;
            so[0] = st.iteration; so[1] = st.evals; so[2] = st.ls_steps; so[3] = st.term;
          }
        }
        __syncwarp();
        rc = __shfl_sync(0xffffffffu, rc, 0);
        if (rc == LM_EVAL) {
          make_class(me.pose, me.cam, &me.cls, lane);
          __syncwarp();
          if (lane == 0) open_pass<CT, P>(sm, me, warp);
        } else {
          state = ST_FETCH;
        }
#ifdef DIB_PASS_TIMING
        if (lane == 0 && a.trace != nullptr && n_rec - 1 < a.trace_cap) {
          double* t = a.trace + ((size_t)me.prob * a.trace_cap + (n_rec - 1)) * kTraceRec;
          const unsigned long long now = global_ns();
          t[13] = (double)(t_complete - t_open);
          t[14] = (double)(now - t_complete);
          t_open = now;
        }
#endif
        continue;
      }
    }
    if (owner < 0) {
      // nothing of mine to do right now (idle, or waiting for helpers to finish my pass): help a CTA-mate
      unsigned m = 0;
      if (lane == 0) m = ld_volatile(&sm.open_mask) & ~(1u << warp);
      m = __shfl_sync(0xffffffffu, m, 0);
      const int o = try_claim(m, k);
      if (o < 0) {
        if (state == ST_IDLE) {
          int na = 0;
          if (lane == 0) na = ld_volatile(&sm.n_active);
          na = __shfl_sync(0xffffffffu, na, 0);
          if (na == 0) {                         // every problem of this CTA is finished
            if (lane == 0) {
              const unsigned long long t_end = global_ns();
              atomicMax(tl + 2, t_end);
              if (blockIdx.x < kCtaEndSlots) atomicMax(cta_end + blockIdx.x, t_end);     // the CTA's last warp wins
            }
            break;
          }
        }
        __nanosleep(state == ST_IDLE ? 400 : 100);
        continue;
      }
      owner = o;
    }
    ProbCtx<CT, P>& oc = sm.ctx[owner];
    {
      const int len = oc.slice_rounds, rounds = oc.rounds;
      r_begin = k * len;
      r_end = min(rounds, r_begin + len);
      if (r_begin > r_end) r_begin = r_end;
    }
    eval_slice<CT, P>(ws, oc, r_begin, r_end, oc.part[k], lane);
    if (lane == 0) {
      __threadfence_block();                      // part[k] before the completion count
      atomicAdd(&oc.done, 1);
    }
  }
}

// Pose matrix from parameters (registration.cpp:161-185).
__device__ void pose_matrix(const double* x, int P, double* M) {
  double aa[3];
  const double* t;
  if (P == 4) { aa[0] = 0; aa[1] = x[0]; aa[2] = 0; t = x + 1; } else { aa[0] = x[0]; aa[1] = x[1]; aa[2] = x[2]; t = x + 3; }
  double R[9];
  const double th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (th2 > DBL_EPSILON) {
    const double th = sqrt(th2);
    const double wx = aa[0] / th, wy = aa[1] / th, wz = aa[2] / th;
    double s, c;
    sincos(th, &s, &c);
    const double omc = 1.0 - c;
    R[0] = c + wx * wx * omc;       R[1] = wx * wy * omc - wz * s;  R[2] = wy * s + wx * wz * omc;
    R[3] = wz * s + wx * wy * omc;  R[4] = c + wy * wy * omc;       R[5] = -wx * s + wy * wz * omc;
    R[6] = -wy * s + wx * wz * omc; R[7] = wx * s + wy * wz * omc;  R[8] = c + wz * wz * omc;
  } else {
    R[0] = 1; R[1] = -aa[2]; R[2] = aa[1];
    R[3] = aa[2]; R[4] = 1; R[5] = -aa[0];
    R[6] = -aa[1]; R[7] = aa[0]; R[8] = 1;
  }
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) M[4 * i + j] = R[3 * i + j]; M[4 * i + 3] = t[i]; }
  M[12] = 0; M[13] = 0; M[14] = 0; M[15] = 1;
}

// Per-sample arg-min over inits (lowest index wins ties; NaN never wins) + pose matrix.
// degenerate (may be NULL): samples without a predicted-inside point get P = I, cost = 1e4 (registration_lsq.py:329-332).
__global__ void frustum_finalize_kernel(const double* params_all, const double* cost_all, int S, int I, int P,
                                        const int32_t* degenerate, double* P16_out, double* cost_out, int32_t* best_out) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  if (degenerate && degenerate[s]) {
    for (int j = 0; j < 16; ++j) P16_out[(size_t)s * 16 + j] = (j % 5 == 0) ? 1.0 : 0.0;
    cost_out[s] = 1e4;
    if (best_out) best_out[s] = 0;
    return;
  }
  int best = 0;
  double bc = cost_all[(size_t)s * I];
  if (!(bc == bc)) bc = INFINITY;
  for (int i = 1; i < I; ++i) {
    const double c = cost_all[(size_t)s * I + i];
    if (c < bc) { bc = c; best = i; }
  }
  pose_matrix(params_all + ((size_t)s * I + best) * 6, P, P16_out + (size_t)s * 16);
  cost_out[s] = cost_all[(size_t)s * I + best];
  if (best_out) best_out[s] = best;
}

// One evaluation pass per sample (test hook and residual-free cost/gradient API): a CTA of kEvalWarps warps takes
// the slices of the sample's pass round-robin and adds the slice sums in slice order -- the same slices, the same
// per-slice arithmetic and the same order as inside the solver, so the totals are bit-identical to the solver's.
constexpr int kEvalWarps = 4;

template <typename CT, int P>
struct EvalSmem {
  WarpScratch<CT, P> scratch[kEvalWarps];
  ProbCtx<CT, P> ctx;
};

template <typename CT, int P>
__global__ void __launch_bounds__(kEvalWarps * 32) frustum_evaluate_kernel(const int32_t* n_pts, int n_stride,
                                                                           const double* K9, const double* x, double H,
                                                                           double W, const float* boxes,
                                                                           const Entry<CT>* packed, int rounds_max,
                                                                           int slice_rounds, int sliced, double* cost_out,
                                                                           double* grad_out, double* JtJ_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  EvalSmem<CT, P>& sm = *reinterpret_cast<EvalSmem<CT, P>*>(smem_raw);
  constexpr int N = NAcc<P>::N;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int s = blockIdx.x;
  ProbCtx<CT, P>& pb = sm.ctx;
  if (tid == 0) {
    const int n = n_pts ? n_pts[s] : n_stride;
    const int rounds = box_rounds(n);
    const int len = sliced ? slice_len(rounds, slice_rounds) : (rounds > 0 ? rounds : 1);
    pb.pk = packed + (size_t)s * rounds_max * kRoundPoints;
    pb.box = boxes + (size_t)s * rounds_max * kBoxRoundFloats;
    pb.rounds = rounds;
    pb.slice_rounds = len;
    pb.nslices = rounds > 0 ? (rounds + len - 1) / len : 1;
    make_cam(K9 + (size_t)s * 9, H, W, &pb.cam);
    make_pose<P>(x + (size_t)s * 6, &pb.pose);
  }
  __syncthreads();
  if (warp == 0) make_class(pb.pose, pb.cam, &pb.cls, lane);
  __syncthreads();
  const int ns = pb.nslices, len = pb.slice_rounds, rounds = pb.rounds;
  for (int k = warp; k < ns; k += kEvalWarps) {
    int r_begin = k * len, r_end = min(rounds, r_begin + len);
    if (r_begin > r_end) r_begin = r_end;
    eval_slice<CT, P>(sm.scratch[warp], pb, r_begin, r_end, pb.part[k], lane);
  }
  __syncthreads();
  if (tid < N) {
    double v = pb.part[0][tid];
    for (int j = 1; j < ns; ++j) v += pb.part[j][tid];
    pb.tot[tid] = v;
  }
  __syncthreads();
  if (tid == 0) {
    cost_out[s] = pb.tot[0];
    for (int j = 0; j < 6; ++j) grad_out[(size_t)s * 6 + j] = (j < P) ? pb.tot[1 + j] : 0.0;
    for (int j = 0; j < 36; ++j) JtJ_out[(size_t)s * 36 + j] = 0.0;
    for (int j = 0; j < P; ++j)
      for (int k = 0; k < P; ++k)
        JtJ_out[(size_t)s * 36 + j * P + k] = pb.tot[1 + P + (j <= k ? tri(P, j, k) : tri(P, k, j))];
  }
}

template <typename CT, int P>
__global__ void frustum_residuals_kernel(const CT* xyz, const int8_t* label, int n, int n_stride, const double* K9,
                                         const double* x, double H, double W, const int32_t* row_offset,
                                         double* residuals) {
  __shared__ PoseConst pc;
  __shared__ Cam cam;
  if (threadIdx.x == 0) { make_cam(K9, H, W, &cam); make_pose<P>(x, &pc); }
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int lab = label[i];
  if (lab != 0 && lab != 1) return;
  double r[3] = {0, 0, 0}, J[3][P];
  int nrows = (lab == 1) ? 3 : 1;
  const bool any = point_rows<P>((double)xyz[i], (double)xyz[n_stride + i], (double)xyz[2 * (size_t)n_stride + i], lab,
                                 cam, pc, r, J, &nrows);
  double s = 0.0;
  for (int k = 0; k < nrows; ++k) s += r[k] * r[k];
  const double sq = sqrt(1.0 / (1.0 + s));
  const int ro = row_offset[i];
  for (int k = 0; k < nrows; ++k) residuals[ro + k] = any ? r[k] * sq : 0.0;
}

// ------------------------------------------------------------------------------------------
// Host side of the C ABI.
// ------------------------------------------------------------------------------------------
static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static size_t box_table_bytes(int S, int n_stride) {
  return align_up((size_t)(S > 0 ? S : 0) * box_rounds(n_stride) * kBoxRoundFloats * sizeof(float), 256);
}
// packed per-launch copy of the clouds; sized for the wider (f64) record so one workspace serves both ABIs
static size_t packed_bytes(int S, int n_stride) {
  return align_up((size_t)(S > 0 ? S : 0) * box_rounds(n_stride) * kRoundPoints * sizeof(Entry<double>), 256);
}

#ifndef DIB_SLICE_AFTER
#define DIB_SLICE_AFTER 48
#endif

static int default_slice_after() {
  static const int v = [] {
    const char* e = getenv("DIB_SLICE_AFTER");           // tuning knob; results depend on it at rounding level only
    const int x = e ? atoi(e) : DIB_SLICE_AFTER;
    return x < 0 ? 0 : x;
  }();
  return v;
}

// Passes of a problem that run as one slice before the fixed slicing starts.  A batch that keeps every warp of the
// machine busy for several waves uses DIB_SLICE_AFTER (only the long solves, i.e. the tail, pay for being helpable); a
// batch with fewer problems than ~4 waves has idle warps from the start, so its passes are sliced from the first one.
// (The two settings give sums that differ at rounding level; a given call is deterministic.)
static int slice_after_for(long long total_problems, long long resident_warps) {
  if (getenv("DIB_SLICE_AFTER")) return default_slice_after();
  return total_problems >= 4 * resident_warps ? default_slice_after() : 0;
}

static int default_slice_rounds();
// Rounds (of 1024 points) per slice.  A small batch (slice_after == 0: idle warps from the start) uses short slices so
// that up to 10 warps can work on one pass of a 20480-point cloud; a large one the default length (fewer slice ends).
static int slice_rounds_for(int slice_after) {
  if (getenv("DIB_SLICE_ROUNDS")) return default_slice_rounds();
  if (slice_after != 0) return default_slice_rounds();
  if (const char* e = getenv("DIB_SMALL_SLICE_ROUNDS")) return atoi(e) > 0 ? atoi(e) : DIB_SMALL_SLICE_ROUNDS;   // tuning knob
  return DIB_SMALL_SLICE_ROUNDS;
}

static int default_slice_rounds() {
  static const int v = [] {
    const char* e = getenv("DIB_SLICE_ROUNDS");          // tuning knob; results depend on it at rounding level only
    const int x = e ? atoi(e) : DIB_SLICE_ROUNDS;
    return x < 1 ? 1 : x;
  }();
  return v;
}

template <typename CT>
static int launch_boxes(const CT* xyz, const int8_t* label, const int32_t* n_pts, int n_stride, int S, float* table,
                        Entry<CT>* packed, cudaStream_t st) {
  const int rounds_max = box_rounds(n_stride);
  if (rounds_max == 0 || S == 0) return DIB_OK;
  DIB_REQUIRE(S <= 65535, "S (%d) exceeds grid.y; split the batch", S);
  const int groups = rounds_max * kRoundGroups;
  dim3 grid((groups + 7) / 8, S);
  static const int interleave = [] { const char* e = getenv("DIB_INTERLEAVE"); return e ? (atoi(e) != 0) : 1; }();   // tuning knob
  frustum_boxes_kernel<CT><<<grid, 256, 0, st>>>(xyz, label, n_pts, n_stride, rounds_max, table, packed, interleave);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

template <typename CT>
static int check_cloud_args(const CT* xyz, const int8_t* label, int n_stride, int S) {
  DIB_REQUIRE(xyz != nullptr && label != nullptr, "xyz/label must not be NULL");
  DIB_REQUIRE(S >= 0 && n_stride >= 0, "negative size");
  DIB_REQUIRE(n_stride % 16 == 0, "n_stride (%d) must be a multiple of 16", n_stride);
  DIB_REQUIRE(((uintptr_t)xyz % 16) == 0 && ((uintptr_t)label % 16) == 0, "xyz/label must be 16-byte aligned");
  return DIB_OK;
}

// Optional CUDA events recorded right before / after the solve kernel on its launch stream (dib_profile_solve_events):
// lets a benchmark time the dominant kernel INSIDE its timed steps instead of in a separate loop.
static thread_local int g_eval_slice_rounds = DIB_SLICE_ROUNDS;   // dib_evaluate_sliced: rounds per slice of frustum_evaluate_* (0 = one piece)
static thread_local void* g_ev_start = nullptr;
static thread_local void* g_ev_stop = nullptr;

// Per-device launch configuration of a solver instantiation, looked up once (cudaFuncSetAttribute and the
// occupancy query cost tens of microseconds per call, which the single-problem drop-in path would pay every time).
struct LaunchCfg { int sms = 0, per_sm = 0, l2_bytes = 0; };
template <typename CT, int P>
static int solver_launch_cfg(LaunchCfg* out) {
  static LaunchCfg cache[64];
  int dev = 0;
  DIB_CHECK_CUDA(cudaGetDevice(&dev));
  if (dev >= 0 && dev < 64 && cache[dev].per_sm > 0) { *out = cache[dev]; return DIB_OK; }
  auto kern = frustum_solve_kernel<CT, P>;
  const size_t smem = sizeof(Smem<CT, P>);
  LaunchCfg c;
  DIB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  DIB_CHECK_CUDA(cudaDeviceGetAttribute(&c.sms, cudaDevAttrMultiProcessorCount, dev));
  DIB_CHECK_CUDA(cudaDeviceGetAttribute(&c.l2_bytes, cudaDevAttrL2CacheSize, dev));
  DIB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c.per_sm, kern, Cfg<CT, P>::kWarps * 32, smem));
  if (c.per_sm < 1) { set_error("solver kernel does not fit an SM (%zu B shared memory)", smem); return DIB_ECUDA; }
  if (dev >= 0 && dev < 64) cache[dev] = c;
  *out = c;
  return DIB_OK;
}

template <typename CT, int P>
static int launch_solve(const SolveArgs& a_in, cudaStream_t st) {
  SolveArgs a = a_in;
  LaunchCfg cfg;
  const int rc = solver_launch_cfg<CT, P>(&cfg);
  if (rc != DIB_OK) return rc;
  constexpr int kW = Cfg<CT, P>::kWarps;
  const long long total = (long long)a.S * a.I;
  if (total < 1) return DIB_OK;
  // One CTA (a team of kW warps, one problem per warp) per SM.  A batch with fewer problems than warps is spread
  // one problem per CTA first (the kernel deals the first wave rank-major), so the spare warps of every CTA help.
  long long grid = (long long)cfg.sms * cfg.per_sm;
  a.slice_after = slice_after_for(total, grid * kW);
  a.slice_rounds = slice_rounds_for(a.slice_after);
  // The last problems of a large batch start while the batch drains: CTA-mates go idle within their first passes, so
  // they are sliced from their first pass on (in the short slices of a small batch) instead of from pass slice_after.
  // "Last" is a queue position, and the queue order is a function of the batch alone: results stay reproducible.
  {
    long long late = a.slice_after > 0 ? grid * kW : 0;
    if (const char* e = getenv("DIB_LATE_PROBLEMS")) late = atoll(e);   // tuning knob
    if (late < 0) late = 0;
    if (late > total) late = total;
    a.late_from = (int)(total - late);
    a.late_slice_rounds = slice_rounds_for(0);
    if (const char* e = getenv("DIB_LATE_SLICE_ROUNDS")) a.late_slice_rounds = atoi(e) > 0 ? atoi(e) : a.late_slice_rounds;
  }

  if (grid > total) grid = total;
  // scheduling chunk: the queue walks chunks of samples rank-major (longest-predicted inits of every sample of the
  // chunk first).  Larger chunks start the long solves earlier (shorter tail); smaller chunks keep the packed clouds
  // of the concurrently running problems inside the L2.  H100 (50 MB L2), 512 x 60 problems of 20480 points, chunk set
  // with DIB_CHUNK_SAMPLES (DESIGN.md 4.3.3): at a 700 W power limit, bench.py's headline (4 steps back to back on two
  // streams, alternating runs) gives 6077-6090 reg/s at 86 samples (28 MB of packed clouds), 6012-6057 at 256 (84 MB),
  // 5950 at 512 (no chunking); at a 400 W limit, 8 steps back to back per value, three interleaved repetitions:
  // 86 samples 107.9 ms per step, 128 (42 MB) 109.2, 171 (56 MB) 111.5, 256 115.5, 512 120.9.  -> aim at 5/8 of the L2
  // per chunk, at least ~2x the resident problems.
  long long chunk = (2 * grid * kW + a.I - 1) / a.I;
  const long long bytes_per_sample = (long long)a.rounds_max * kRoundPoints * (long long)sizeof(Entry<CT>);
  const long long chunk_bytes = (long long)cfg.l2_bytes * 5 / 8;
  if (bytes_per_sample > 0 && chunk < chunk_bytes / bytes_per_sample) chunk = chunk_bytes / bytes_per_sample;
  if (const char* e = getenv("DIB_CHUNK_SAMPLES")) chunk = atoll(e);   // tuning knob
  if (chunk < 1) chunk = 1;
  if (chunk > a.S) chunk = a.S;
  {
    // equal-sized chunks: a short last chunk would bring the tail back
    const long long nchunks = (a.S + chunk - 1) / chunk;
    chunk = (a.S + nchunks - 1) / nchunks;
  }
  a.chunk = (int)chunk;
  if (g_ev_start) DIB_CHECK_CUDA(cudaEventRecord((cudaEvent_t)g_ev_start, st));
  frustum_solve_kernel<CT, P><<<(unsigned)grid, kW * 32, sizeof(Smem<CT, P>), st>>>(a);
  DIB_CHECK_CUDA(cudaGetLastError());
  if (g_ev_stop) DIB_CHECK_CUDA(cudaEventRecord((cudaEvent_t)g_ev_stop, st));
  return DIB_OK;
}

static size_t solve_workspace_bytes_impl(int S, int I, int n_stride) {
  const size_t n = (size_t)(S > 0 ? S : 0) * (size_t)(I > 0 ? I : 0);
  return kHeaderBytes + align_up(n * 6 * sizeof(double), 256) + align_up(n * sizeof(double), 256) +
         align_up(n * 4 * sizeof(int32_t), 256) + box_table_bytes(S, n_stride > 0 ? n_stride : 0) +
         packed_bytes(S, n_stride > 0 ? n_stride : 0) + align_up(n * sizeof(int32_t), 256);
}

template <typename CT>
static int solve_batch(const CT* xyz, const int8_t* label, const int32_t* n_pts, int n_stride, const double* K9,
                       const double* init, const double* lb3, const double* ub3, double H, double W, int max_iter,
                       int is_2d, int S, int I, double* P16_out, double* cost_out, int32_t* best_out,
                       double* params_all, double* cost_all, int32_t* stats_all, const int32_t* degenerate,
                       double* trace, int trace_cap, void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  int rc = check_cloud_args<CT>(xyz, label, n_stride, S);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(I >= 1, "I must be >= 1");
  DIB_REQUIRE(K9 && init && lb3 && ub3 && P16_out && cost_out, "NULL argument");
  DIB_REQUIRE((long long)S * I < (1ll << 30), "S*I too large");
  DIB_REQUIRE(trace == nullptr || trace_cap >= 1, "trace_cap must be >= 1");
  if (S == 0) return DIB_OK;
  if (workspace_bytes < solve_workspace_bytes_impl(S, I, n_stride) || workspace == nullptr) {
    set_error("workspace too small: %zu < %zu", workspace_bytes, solve_workspace_bytes_impl(S, I, n_stride));
    return DIB_ENOMEM;
  }
  DIB_REQUIRE(((uintptr_t)workspace % 256) == 0, "workspace must be 256-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* ws = (unsigned char*)workspace;
  const size_t n = (size_t)S * I;
  SolveArgs a;
  a.queue = (unsigned int*)ws;
  size_t off = kHeaderBytes;
  a.params_all = params_all ? params_all : (double*)(ws + off);
  off += align_up(n * 6 * sizeof(double), 256);
  a.cost_all = cost_all ? cost_all : (double*)(ws + off);
  off += align_up(n * sizeof(double), 256);
  a.stats_all = stats_all ? stats_all : (int32_t*)(ws + off);
  off += align_up(n * 4 * sizeof(int32_t), 256);
  float* table = (float*)(ws + off);
  off += box_table_bytes(S, n_stride);
  Entry<CT>* packed = (Entry<CT>*)(ws + off);
  off += packed_bytes(S, n_stride);
  int32_t* perm = (int32_t*)(ws + off);
  a.boxes = table;
  a.packed = packed;
  a.rounds_max = box_rounds(n_stride);
  a.perm = perm;
  a.xyz = xyz; a.label = label; a.n_pts = n_pts; a.n_stride = n_stride; a.K9 = K9; a.init = init;
  for (int k = 0; k < 3; ++k) { a.lb[k] = lb3[k]; a.ub[k] = ub3[k]; }
  a.H = H; a.W = W; a.max_iter = max_iter; a.S = S; a.I = I;
  a.chunk = 1;
  a.slice_rounds = default_slice_rounds();
  a.slice_after = 0;                                   // decided in launch_solve (needs the grid)
  a.late_from = 0x7fffffff; a.late_slice_rounds = a.slice_rounds;
  a.trace = trace; a.trace_cap = trace_cap;
  DIB_CHECK_CUDA(cudaMemsetAsync(a.queue, 0, kHeaderBytes, st));
  DIB_CHECK_CUDA(cudaMemsetAsync((unsigned char*)a.queue + 8, 0xff, 16, st));   // timeline minima start at ~0ull
  if (trace) DIB_CHECK_CUDA(cudaMemsetAsync(trace, 0, n * (size_t)trace_cap * kTraceRec * sizeof(double), st));
  rc = launch_boxes<CT>(xyz, label, n_pts, n_stride, S, table, packed, st);
  if (rc != DIB_OK) return rc;
  {
    const int threads = I < 256 ? ((I + 31) / 32) * 32 : 256;
    DIB_REQUIRE((size_t)I * sizeof(double) <= 48 * 1024, "I=%d too large for the ordering kernel", I);
    frustum_order_kernel<<<S, threads, (size_t)I * sizeof(double), st>>>(init, I, perm);
    DIB_CHECK_CUDA(cudaGetLastError());
  }
  rc = is_2d ? launch_solve<CT, 4>(a, st) : launch_solve<CT, 6>(a, st);
  if (rc != DIB_OK) return rc;
  frustum_finalize_kernel<<<(S + 127) / 128, 128, 0, st>>>(a.params_all, a.cost_all, S, I, is_2d ? 4 : 6, degenerate,
                                                          P16_out, cost_out, best_out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

template <typename CT, int P>
static int launch_evaluate(const int32_t* n_pts, int n_stride, const double* K9, const double* x, double H, double W,
                           int S, const float* table, const Entry<CT>* packed, double* cost_out, double* grad_out,
                           double* JtJ_out, cudaStream_t st) {
  auto kern = frustum_evaluate_kernel<CT, P>;
  const size_t smem = sizeof(EvalSmem<CT, P>);
  static bool configured[64] = {};
  int dev = 0;
  DIB_CHECK_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !configured[dev]) {
    DIB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (dev >= 0 && dev < 64) configured[dev] = true;
  }
  kern<<<S, kEvalWarps * 32, smem, st>>>(n_pts, n_stride, K9, x, H, W, table, packed, box_rounds(n_stride),
                                         g_eval_slice_rounds > 0 ? g_eval_slice_rounds : 1, g_eval_slice_rounds > 0 ? 1 : 0, cost_out,
                                         grad_out, JtJ_out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

template <typename CT>
static int evaluate_batch(const CT* xyz, const int8_t* label, const int32_t* n_pts, int n_stride, const double* K9,
                          const double* x, double H, double W, int is_2d, int S, double* cost_out, double* grad_out,
                          double* JtJ_out, void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  int rc = check_cloud_args<CT>(xyz, label, n_stride, S);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(K9 && x && cost_out && grad_out && JtJ_out, "NULL argument");
  if (S == 0) return DIB_OK;
  if (workspace_bytes < frustum_evaluate_workspace_bytes(S, n_stride) || workspace == nullptr) {
    set_error("workspace too small: %zu < %zu", workspace_bytes, frustum_evaluate_workspace_bytes(S, n_stride));
    return DIB_ENOMEM;
  }
  DIB_REQUIRE(((uintptr_t)workspace % 256) == 0, "workspace must be 256-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  float* table = (float*)workspace;
  Entry<CT>* packed = (Entry<CT>*)((unsigned char*)workspace + box_table_bytes(S, n_stride));
  rc = launch_boxes<CT>(xyz, label, n_pts, n_stride, S, table, packed, st);
  if (rc != DIB_OK) return rc;
  return is_2d ? launch_evaluate<CT, 4>(n_pts, n_stride, K9, x, H, W, S, table, packed, cost_out, grad_out, JtJ_out, st)
               : launch_evaluate<CT, 6>(n_pts, n_stride, K9, x, H, W, S, table, packed, cost_out, grad_out, JtJ_out, st);
}

template <typename CT>
static int residuals_single(const CT* xyz, const int8_t* label, int n, int n_stride, const double* K9,
                            const double* x, double H, double W, int is_2d, const int32_t* row_offset,
                            double* residuals, dib_stream_t stream) {
  DIB_REQUIRE(xyz && label && K9 && x && residuals, "NULL argument");
  DIB_REQUIRE(n >= 0 && n <= n_stride, "bad n");
  if (n == 0) return DIB_OK;                            // no rows: the (empty) row offsets may be NULL
  DIB_REQUIRE(row_offset, "NULL argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int blocks = (n + 255) / 256;
  if (is_2d)
    frustum_residuals_kernel<CT, 4><<<blocks, 256, 0, st>>>(xyz, label, n, n_stride, K9, x, H, W, row_offset, residuals);
  else
    frustum_residuals_kernel<CT, 6><<<blocks, 256, 0, st>>>(xyz, label, n, n_stride, K9, x, H, W, row_offset, residuals);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // namespace dib

extern "C" {

int dib_abi_version(void) { return 4; }
const char* dib_last_error(void) { return dib::g_err; }

void dib_evaluate_sliced(int rounds_per_slice) { dib::g_eval_slice_rounds = rounds_per_slice < 0 ? 0 : rounds_per_slice; }

int frustum_solve_slice_after(int S, int I, int is_2d, int f64_record) {
  dib::LaunchCfg cfg;
  int rc;
  int kw;
  if (f64_record) { rc = is_2d ? dib::solver_launch_cfg<double, 4>(&cfg) : dib::solver_launch_cfg<double, 6>(&cfg);
                    kw = is_2d ? dib::Cfg<double, 4>::kWarps : dib::Cfg<double, 6>::kWarps; }
  else { rc = is_2d ? dib::solver_launch_cfg<float, 4>(&cfg) : dib::solver_launch_cfg<float, 6>(&cfg);
         kw = is_2d ? dib::Cfg<float, 4>::kWarps : dib::Cfg<float, 6>::kWarps; }
  if (rc != DIB_OK) return rc;
  return dib::slice_after_for((long long)S * I, (long long)cfg.sms * cfg.per_sm * kw);
}

int frustum_solve_slice_rounds(int S, int I, int is_2d, int f64_record) {
  const int after = frustum_solve_slice_after(S, I, is_2d, f64_record);
  return after < 0 ? after : dib::slice_rounds_for(after);
}

void dib_profile_solve_events(void* start_event, void* stop_event) {
  dib::g_ev_start = start_event;
  dib::g_ev_stop = stop_event;
}

int dib_device_sm_count(void) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return DIB_ENODEV;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return DIB_ENODEV;
  return sms;
}

size_t frustum_solve_workspace_bytes(int S, int I, int n_stride) { return dib::solve_workspace_bytes_impl(S, I, n_stride); }

size_t frustum_evaluate_workspace_bytes(int S, int n_stride) {
  return dib::box_table_bytes(S, n_stride > 0 ? n_stride : 0) + dib::packed_bytes(S, n_stride > 0 ? n_stride : 0) + 256;
}

int frustum_solve_batch_f32(const float* xyz, const int8_t* label, const int32_t* n_pts, int n_stride,
                            const double* K9, const double* init, const double* lb3, const double* ub3, double H,
                            double W, int max_iter, int is_2d, int S, int I, double* P16_out, double* cost_out,
                            int32_t* best_out, double* params_all, double* cost_all, int32_t* stats_all,
                            void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  return dib::solve_batch<float>(xyz, label, n_pts, n_stride, K9, init, lb3, ub3, H, W, max_iter, is_2d, S, I,
                                 P16_out, cost_out, best_out, params_all, cost_all, stats_all, nullptr, nullptr, 0,
                                 workspace, workspace_bytes, stream);
}

int frustum_solve_batch_f64(const double* xyz, const int8_t* label, const int32_t* n_pts, int n_stride,
                            const double* K9, const double* init, const double* lb3, const double* ub3, double H,
                            double W, int max_iter, int is_2d, int S, int I, double* P16_out, double* cost_out,
                            int32_t* best_out, double* params_all, double* cost_all, int32_t* stats_all,
                            void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  return dib::solve_batch<double>(xyz, label, n_pts, n_stride, K9, init, lb3, ub3, H, W, max_iter, is_2d, S, I,
                                  P16_out, cost_out, best_out, params_all, cost_all, stats_all, nullptr, nullptr, 0,
                                  workspace, workspace_bytes, stream);
}

int frustum_solve_traced_f32(const float* xyz, const int8_t* label, const int32_t* n_pts, int n_stride,
                             const double* K9, const double* init, const double* lb3, const double* ub3, double H,
                             double W, int max_iter, int is_2d, int S, int I, double* P16_out, double* cost_out,
                             int32_t* best_out, double* params_all, double* cost_all, int32_t* stats_all,
                             double* trace, int trace_cap, void* workspace, size_t workspace_bytes,
                             dib_stream_t stream) {
  DIB_REQUIRE(trace != nullptr, "trace must not be NULL");
  return dib::solve_batch<float>(xyz, label, n_pts, n_stride, K9, init, lb3, ub3, H, W, max_iter, is_2d, S, I,
                                 P16_out, cost_out, best_out, params_all, cost_all, stats_all, nullptr, trace,
                                 trace_cap, workspace, workspace_bytes, stream);
}

// Whole per-sample body of registration_lsq.py:329-343 in one call: initial guess + front filter + perturbed inits
// (frustum_prepare_batch_f32), the multi-start solve, the arg-min and the degenerate-sample rule.
static size_t register_front_bytes(int S, int I, int n_in, size_t off[6]) {
  const size_t Ns = (size_t)((n_in > 0 ? n_in : 0) + 15) & ~(size_t)15;
  const size_t s = (size_t)(S > 0 ? S : 0), i = (size_t)(I > 0 ? I : 0);
  size_t o = 0;
  off[0] = o; o += dib::align_up(s * 3 * Ns * sizeof(float), 256);      // xyz
  off[1] = o; o += dib::align_up(s * Ns, 256);                          // label
  off[2] = o; o += dib::align_up(s * sizeof(int32_t), 256);             // n_pts
  off[3] = o; o += dib::align_up(s * i * 4 * sizeof(double), 256);      // init
  off[4] = o; o += dib::align_up(s * sizeof(double), 256);              // init_y_angle
  off[5] = o; o += dib::align_up(s * sizeof(int32_t), 256);             // degenerate
  return o;
}

size_t frustum_register_workspace_bytes(int S, int I, int n_in) {
  size_t off[6];
  const int Ns = ((n_in > 0 ? n_in : 0) + 15) & ~15;
  return register_front_bytes(S, I, n_in, off) + dib::solve_workspace_bytes_impl(S, I, Ns);
}

int frustum_register_batch_f32(const float* xyz_in, const int8_t* pred, int n_in, int n_in_stride, int S, int I,
                               uint64_t seed, double ry_sigma, double t_amp, const double* K9, const double* lb3,
                               const double* ub3, double H, double W, int max_iter, int is_2d, double* P16_out,
                               double* cost_out, int32_t* best_out, double* init_y_angle_out, int32_t* n_pts_out,
                               int32_t* degenerate_out, double* init_out, double* params_all, double* cost_all,
                               int32_t* stats_all, void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  DIB_REQUIRE(S >= 0 && I >= 1 && n_in >= 0, "bad sizes");
  if (S == 0) return DIB_OK;
  size_t off[6];
  const size_t front = register_front_bytes(S, I, n_in, off);
  const int Ns = (n_in + 15) & ~15;
  const size_t need = front + dib::solve_workspace_bytes_impl(S, I, Ns);
  if (workspace == nullptr || workspace_bytes < need) {
    dib::set_error("workspace too small: %zu < %zu", workspace_bytes, need);
    return DIB_ENOMEM;
  }
  DIB_REQUIRE(((uintptr_t)workspace % 256) == 0, "workspace must be 256-byte aligned");
  unsigned char* ws = (unsigned char*)workspace;
  float* xyz = (float*)(ws + off[0]);
  int8_t* label = (int8_t*)(ws + off[1]);
  int32_t* n_pts = n_pts_out ? n_pts_out : (int32_t*)(ws + off[2]);
  double* init = init_out ? init_out : (double*)(ws + off[3]);
  double* ang = init_y_angle_out ? init_y_angle_out : (double*)(ws + off[4]);
  int32_t* degen = degenerate_out ? degenerate_out : (int32_t*)(ws + off[5]);
  int rc = frustum_prepare_batch_f32(xyz_in, pred, n_in, n_in_stride, S, I, seed, ry_sigma, t_amp, 1, xyz, label, n_pts,
                                     init, ang, degen, nullptr, 0, stream);
  if (rc != DIB_OK) return rc;
  return dib::solve_batch<float>(xyz, label, n_pts, Ns, K9, init, lb3, ub3, H, W, max_iter, is_2d, S, I, P16_out,
                                 cost_out, best_out, params_all, cost_all, stats_all, degen, nullptr, 0, ws + front,
                                 workspace_bytes - front, stream);
}

int frustum_evaluate_f32(const float* xyz, const int8_t* label, const int32_t* n_pts, int n_stride, const double* K9,
                         const double* x, double H, double W, int is_2d, int S, double* cost_out, double* grad_out,
                         double* JtJ_out, void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  return dib::evaluate_batch<float>(xyz, label, n_pts, n_stride, K9, x, H, W, is_2d, S, cost_out, grad_out, JtJ_out,
                                    workspace, workspace_bytes, stream);
}
int frustum_evaluate_f64(const double* xyz, const int8_t* label, const int32_t* n_pts, int n_stride,
                         const double* K9, const double* x, double H, double W, int is_2d, int S, double* cost_out,
                         double* grad_out, double* JtJ_out, void* workspace, size_t workspace_bytes,
                         dib_stream_t stream) {
  return dib::evaluate_batch<double>(xyz, label, n_pts, n_stride, K9, x, H, W, is_2d, S, cost_out, grad_out, JtJ_out,
                                     workspace, workspace_bytes, stream);
}

int frustum_residuals_f32(const float* xyz, const int8_t* label, int n, int n_stride, const double* K9,
                          const double* x, double H, double W, int is_2d, const int32_t* row_offset,
                          double* residuals, dib_stream_t stream) {
  return dib::residuals_single<float>(xyz, label, n, n_stride, K9, x, H, W, is_2d, row_offset, residuals, stream);
}
int frustum_residuals_f64(const double* xyz, const int8_t* label, int n, int n_stride, const double* K9,
                          const double* x, double H, double W, int is_2d, const int32_t* row_offset,
                          double* residuals, dib_stream_t stream) {
  return dib::residuals_single<double>(xyz, label, n, n_stride, K9, x, H, W, is_2d, row_offset, residuals, stream);
}

}  // extern "C"
