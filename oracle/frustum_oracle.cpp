// =====================================================================================
// TEST INFRASTRUCTURE ONLY -- CPU oracle for the inverse-camera-projection registration
// solver.  Nothing under oracle/ is ever imported, linked or executed by the product
// path (deepi2p_b200/); only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline
// legs may use it.
//
// PARITY UNPINNED: the reference solver (evaluation/frustum_reg/src/registration.cpp)
// delegates all arithmetic to Ceres Solver (un-vendored, unpinned; era 1.14 / 2.0) and
// Eigen, neither of which exists in this container, and the reference ships no golden
// vectors or asserting tests for this path (SURVEY.md section 4, 8c).  This file restates
//   * the reference's own residual functors, parameter layout, bounds, loss and outputs
//     (cited per function below), evaluated with forward-mode dual numbers exactly the
//     way Ceres' AutoDiffCostFunction would (so it is an independent check of the
//     analytic derivatives the CUDA kernels use), and
//   * Ceres' published trust-region algorithm with the options the reference selects
//     (TRUST_REGION + LEVENBERG_MARQUARDT, DENSE_QR, Jacobi scaling, CauchyLoss(1.0),
//     box bounds -> projected Armijo line search with cubic interpolation, monotonic
//     steps, default tolerances) from its documentation / memory of
//     trust_region_minimizer.cc, levenberg_marquardt_strategy.cc, dense_qr_solver.cc,
//     corrector.cc, loss_function.cc, line_search.cc, polynomial.cc, parameter_block.h.
// Known deliberate deviation: roots of the degree-4 derivative polynomial in the 3-sample
// line-search interpolation are found by (total-step) Durand-Kerner iteration instead of companion
// matrix eigenvalues (same roots, different rounding).
//
// Build: g++ -O2 -shared -fPIC -std=c++17 (see oracle/build.py).  C ABI at the bottom.
// =====================================================================================
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <complex>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

namespace {

// ---------------------------------------------------------------------------
// Dual numbers (value + N partials), arithmetic rules as in Ceres' jet.h.
// ---------------------------------------------------------------------------
template <int N>
struct Dual {
  double a;
  double v[N];
  Dual() : a(0.0) { for (int i = 0; i < N; ++i) v[i] = 0.0; }
  explicit Dual(double s) : a(s) { for (int i = 0; i < N; ++i) v[i] = 0.0; }
  Dual(double s, int k) : a(s) { for (int i = 0; i < N; ++i) v[i] = 0.0; v[k] = 1.0; }
};

template <int N> Dual<N> operator-(const Dual<N>& f) {
  Dual<N> r; r.a = -f.a; for (int i = 0; i < N; ++i) r.v[i] = -f.v[i]; return r;
}
template <int N> Dual<N> operator+(const Dual<N>& f, const Dual<N>& g) {
  Dual<N> r; r.a = f.a + g.a; for (int i = 0; i < N; ++i) r.v[i] = f.v[i] + g.v[i]; return r;
}
template <int N> Dual<N> operator+(const Dual<N>& f, double s) { Dual<N> r = f; r.a = f.a + s; return r; }
template <int N> Dual<N> operator-(const Dual<N>& f, const Dual<N>& g) {
  Dual<N> r; r.a = f.a - g.a; for (int i = 0; i < N; ++i) r.v[i] = f.v[i] - g.v[i]; return r;
}
template <int N> Dual<N> operator*(const Dual<N>& f, const Dual<N>& g) {
  Dual<N> r; r.a = f.a * g.a; for (int i = 0; i < N; ++i) r.v[i] = f.a * g.v[i] + f.v[i] * g.a; return r;
}
template <int N> Dual<N> operator*(const Dual<N>& f, double s) {
  Dual<N> r; r.a = f.a * s; for (int i = 0; i < N; ++i) r.v[i] = f.v[i] * s; return r;
}
template <int N> Dual<N> operator*(double s, const Dual<N>& f) { return f * s; }
template <int N> Dual<N> operator/(const Dual<N>& f, const Dual<N>& g) {
  // (a+u)/(b+v) = a/b + (u - (a/b) v)/b
  const double g_inv = 1.0 / g.a;
  const double q = f.a * g_inv;
  Dual<N> r; r.a = q; for (int i = 0; i < N; ++i) r.v[i] = (f.v[i] - q * g.v[i]) * g_inv; return r;
}
template <int N> Dual<N> operator/(double s, const Dual<N>& g) {
  const double m = -s / (g.a * g.a);
  Dual<N> r; r.a = s / g.a; for (int i = 0; i < N; ++i) r.v[i] = g.v[i] * m; return r;
}
template <int N> bool operator<(const Dual<N>& f, const Dual<N>& g) { return f.a < g.a; }
template <int N> bool operator>(const Dual<N>& f, const Dual<N>& g) { return f.a > g.a; }
template <int N> Dual<N> dsqrt(const Dual<N>& f) {
  const double t = std::sqrt(f.a); const double k = 1.0 / (2.0 * t);
  Dual<N> r; r.a = t; for (int i = 0; i < N; ++i) r.v[i] = f.v[i] * k; return r;
}
template <int N> Dual<N> dcos(const Dual<N>& f) {
  const double c = std::cos(f.a), s = std::sin(f.a);
  Dual<N> r; r.a = c; for (int i = 0; i < N; ++i) r.v[i] = -s * f.v[i]; return r;
}
template <int N> Dual<N> dsin(const Dual<N>& f) {
  const double c = std::cos(f.a), s = std::sin(f.a);
  Dual<N> r; r.a = s; for (int i = 0; i < N; ++i) r.v[i] = c * f.v[i]; return r;
}
// abs keeps x for x >= 0 (sgn(0) = +1); fmax(x, y) keeps x on ties.
template <int N> Dual<N> dabs(const Dual<N>& f) { return f.a < 0.0 ? -f : f; }
template <int N> Dual<N> dfmax(const Dual<N>& x, const Dual<N>& y) { return x < y ? y : x; }

// ---------------------------------------------------------------------------
// Rotation of a point by an angle-axis vector (Rodrigues; first-order branch when
// |aa|^2 <= DBL_EPSILON).  Follows the call sites registration_3d.hpp:40,111 and
// registration_2d.hpp:40-41,112-113 (ceres::AngleAxisRotatePoint).
// ---------------------------------------------------------------------------
template <int N>
void rotate_point(const Dual<N> aa[3], const double pt[3], Dual<N> out[3]) {
  const Dual<N> theta2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (theta2.a > std::numeric_limits<double>::epsilon()) {
    const Dual<N> theta = dsqrt(theta2);
    const Dual<N> ct = dcos(theta), st = dsin(theta);
    const Dual<N> tinv = 1.0 / theta;
    const Dual<N> w[3] = {aa[0] * tinv, aa[1] * tinv, aa[2] * tinv};
    const Dual<N> wxp[3] = {w[1] * pt[2] - w[2] * pt[1],
                            w[2] * pt[0] - w[0] * pt[2],
                            w[0] * pt[1] - w[1] * pt[0]};
    const Dual<N> one_m_ct = -(ct + (-1.0));   // 1 - cos(theta)
    const Dual<N> tmp = (w[0] * pt[0] + w[1] * pt[1] + w[2] * pt[2]) * one_m_ct;
    for (int k = 0; k < 3; ++k) out[k] = ct * pt[k] + wxp[k] * st + w[k] * tmp;
  } else {
    const Dual<N> wxp[3] = {aa[1] * pt[2] - aa[2] * pt[1],
                            aa[2] * pt[0] - aa[0] * pt[2],
                            aa[0] * pt[1] - aa[1] * pt[0]};
    for (int k = 0; k < 3; ++k) out[k] = wxp[k] + pt[k];
  }
}

struct Camera { double fx, fy, cx, cy, H1, W1; };

// q = R p + t for the 2-D (4 params: ry,tx,ty,tz) or 3-D (6 params: aa,t) layout.
// registration.cpp:24-50 (layout), registration_{2d,3d}.hpp:38-46 / 110-118 (transform).
template <int N>
void transform_point(const double* x, const double pt[3], Dual<N> q[3]) {
  Dual<N> aa[3];
  int toff;
  if (N == 4) { aa[0] = Dual<N>(0.0); aa[1] = Dual<N>(x[0], 0); aa[2] = Dual<N>(0.0); toff = 1; }
  else { for (int k = 0; k < 3; ++k) aa[k] = Dual<N>(x[k], k); toff = 3; }
  rotate_point<N>(aa, pt, q);
  for (int k = 0; k < 3; ++k) q[k] = q[k] + Dual<N>(x[toff + k], toff + k);
}

// label 0 -- "point should project OUTSIDE the image": one residual row.
// registration_3d.hpp:34-68, registration_2d.hpp:34-69.
template <int N>
void residual_outside(const double* x, const double pt[3], const Camera& c, Dual<N> r[1]) {
  Dual<N> q[3];
  transform_point<N>(x, pt, q);
  const Dual<N> px = (c.fx * q[0]) / q[2] + c.cx;
  const Dual<N> py = (c.fy * q[1]) / q[2] + c.cy;
  const Dual<N> zero(0.0);
  const Dual<N> xd = Dual<N>(c.W1 * 0.5) - dabs(px + (-(c.W1 * 0.5)));
  const Dual<N> is_x_in = dfmax(xd, zero) / xd;
  const Dual<N> yd = Dual<N>(c.H1 * 0.5) - dabs(py + (-(c.H1 * 0.5)));
  const Dual<N> is_y_in = dfmax(yd, zero) / yd;
  const Dual<N> is_front = dfmax(q[2], zero) / q[2];
  const Dual<N> xy = xd + yd;
  r[0] = ((xy * is_front) * is_x_in) * is_y_in;
}

// label 1 -- "point should project INSIDE the image": three residual rows.
// registration_3d.hpp:105-127, registration_2d.hpp:106-129.
template <int N>
void residual_inside(const double* x, const double pt[3], const Camera& c, Dual<N> r[3]) {
  Dual<N> q[3];
  transform_point<N>(x, pt, q);
  const Dual<N> px = (c.fx * q[0]) / q[2] + c.cx;
  const Dual<N> py = (c.fy * q[1]) / q[2] + c.cy;
  const Dual<N> zero(0.0);
  r[0] = dfmax(-px, zero) + dfmax(px + (-c.W1), zero);
  r[1] = dfmax(-py, zero) + dfmax(py + (-c.H1), zero);
  r[2] = dfmax(-q[2], zero) * 100.0;
}

// ---------------------------------------------------------------------------
// Problem = the residual blocks registration.cpp:87-125 adds, in point order.
// ---------------------------------------------------------------------------
struct Problem {
  const double* px; const double* py; const double* pz;   // N each
  const int32_t* label;
  int64_t n;
  Camera cam;
  int P;            // 4 or 6
  int toff;         // 1 or 3
  double lb[6], ub[6];
  int64_t rows;     // n0 + 3 n1
};

struct Eval {
  double cost;
  std::vector<double> r;    // corrected residuals, rows
  std::vector<double> J;    // corrected jacobian, rows x P row-major (only if want_jac)
  double g[6];              // J^T r (only if want_jac)
};

// One pass over all residual blocks: cost = sum 0.5*rho(s), rho = log(1+s) (CauchyLoss(1.0),
// registration.cpp:103,121); residuals and Jacobian rows scaled by sqrt(rho'(s)) (Ceres
// corrector, rho'' < 0 branch).
template <int N>
void evaluate_impl(const Problem& pb, const double* x, bool want_jac, bool want_res, Eval* out) {
  double cost = 0.0;
  if (want_res || want_jac) out->r.assign(pb.rows, 0.0);
  if (want_jac) { out->J.assign(pb.rows * N, 0.0); for (int j = 0; j < 6; ++j) out->g[j] = 0.0; }
  int64_t row = 0;
  for (int64_t i = 0; i < pb.n; ++i) {
    const int lab = pb.label[i];
    if (lab != 0 && lab != 1) continue;
    const double pt[3] = {pb.px[i], pb.py[i], pb.pz[i]};
    Dual<N> r[3];
    const int nr = (lab == 1) ? 3 : 1;
    if (lab == 1) residual_inside<N>(x, pt, pb.cam, r); else residual_outside<N>(x, pt, pb.cam, r);
    double s = 0.0;
    for (int k = 0; k < nr; ++k) s += r[k].a * r[k].a;
    const double sum = 1.0 + s;
    const double inv = 1.0 / sum;
    const double rho0 = std::log(sum);
    const double rho1 = std::max(std::numeric_limits<double>::min(), inv);
    cost += 0.5 * rho0;
    if (want_res || want_jac) {
      const double sq = std::sqrt(rho1);
      for (int k = 0; k < nr; ++k) {
        if (want_jac) {
          for (int j = 0; j < N; ++j) out->J[(row + k) * N + j] = r[k].v[j] * sq;
        }
        out->r[row + k] = r[k].a * sq;
      }
      if (want_jac) {
        for (int k = 0; k < nr; ++k)
          for (int j = 0; j < N; ++j) out->g[j] += out->J[(row + k) * N + j] * out->r[row + k];
      }
    }
    row += nr;
  }
  out->cost = cost;
}

void evaluate(const Problem& pb, const double* x, bool want_jac, bool want_res, Eval* out) {
  if (pb.P == 4) evaluate_impl<4>(pb, x, want_jac, want_res, out);
  else evaluate_impl<6>(pb, x, want_jac, want_res, out);
}

// x (+) delta followed by projection on the box (Ceres ParameterBlock::Plus).
void plus_project(const Problem& pb, const double* x, const double* d, double* out) {
  for (int j = 0; j < pb.P; ++j) {
    double v = x[j] + d[j];
    v = std::max(v, pb.lb[j]);
    v = std::min(v, pb.ub[j]);
    out[j] = v;
  }
}

// ---------------------------------------------------------------------------
// Dense least squares min || A y - b ||, A (m x n) row-major, by Householder QR
// (DENSE_QR, registration.cpp:138).  Overwrites A and b.  Returns false on a zero pivot.
// ---------------------------------------------------------------------------
bool householder_lstsq(std::vector<double>& A, std::vector<double>& b, int64_t m, int n, double* y) {
  std::vector<double> diagR(n);
  for (int k = 0; k < n; ++k) {
    double norm2 = 0.0;
    for (int64_t i = k; i < m; ++i) norm2 += A[i * n + k] * A[i * n + k];
    const double norm = std::sqrt(norm2);
    if (norm == 0.0) { diagR[k] = 0.0; continue; }
    const double akk = A[k * n + k];
    const double alpha = (akk > 0.0) ? -norm : norm;
    // v = a_k - alpha e_k ; stored in place
    A[k * n + k] = akk - alpha;
    double vnorm2 = norm2 - akk * akk + A[k * n + k] * A[k * n + k];
    if (vnorm2 == 0.0) { diagR[k] = alpha; continue; }
    for (int j = k + 1; j < n; ++j) {
      double dot = 0.0;
      for (int64_t i = k; i < m; ++i) dot += A[i * n + k] * A[i * n + j];
      const double f = 2.0 * dot / vnorm2;
      for (int64_t i = k; i < m; ++i) A[i * n + j] -= f * A[i * n + k];
    }
    {
      double dot = 0.0;
      for (int64_t i = k; i < m; ++i) dot += A[i * n + k] * b[i];
      const double f = 2.0 * dot / vnorm2;
      for (int64_t i = k; i < m; ++i) b[i] -= f * A[i * n + k];
    }
    diagR[k] = alpha;
  }
  for (int k = n - 1; k >= 0; --k) {
    double s = b[k];
    for (int j = k + 1; j < n; ++j) s -= A[k * n + j] * y[j];
    if (diagR[k] == 0.0) return false;
    y[k] = s / diagR[k];
  }
  return true;
}

// ---------------------------------------------------------------------------
// Line-search support (Ceres line_search.cc / polynomial.cc semantics).
// ---------------------------------------------------------------------------
struct Sample { double x, value, gradient; bool value_valid, gradient_valid; };

// Solve a small dense system with full pivoting (FullPivLU, threshold 0).
bool solve_full_pivot(int n, std::vector<double> M, std::vector<double> rhs, double* sol) {
  std::vector<int> colperm(n);
  for (int i = 0; i < n; ++i) colperm[i] = i;
  for (int k = 0; k < n; ++k) {
    int pr = k, pc = k; double best = -1.0;
    for (int i = k; i < n; ++i) for (int j = k; j < n; ++j)
      if (std::fabs(M[i * n + j]) > best) { best = std::fabs(M[i * n + j]); pr = i; pc = j; }
    if (best == 0.0) { for (int i = k; i < n; ++i) rhs[i] = 0.0; break; }
    if (pr != k) { for (int j = 0; j < n; ++j) std::swap(M[pr * n + j], M[k * n + j]); std::swap(rhs[pr], rhs[k]); }
    if (pc != k) { for (int i = 0; i < n; ++i) std::swap(M[i * n + pc], M[i * n + k]); std::swap(colperm[pc], colperm[k]); }
    for (int i = k + 1; i < n; ++i) {
      const double f = M[i * n + k] / M[k * n + k];
      for (int j = k; j < n; ++j) M[i * n + j] -= f * M[k * n + j];
      rhs[i] -= f * rhs[k];
    }
  }
  std::vector<double> z(n, 0.0);
  for (int k = n - 1; k >= 0; --k) {
    if (M[k * n + k] == 0.0) { z[k] = 0.0; continue; }
    double s = rhs[k];
    for (int j = k + 1; j < n; ++j) s -= M[k * n + j] * z[j];
    z[k] = s / M[k * n + k];
  }
  for (int k = 0; k < n; ++k) sol[colperm[k]] = z[k];
  return true;
}

double poly_eval(const std::vector<double>& p, double x) {   // highest degree first
  double v = 0.0;
  for (double c : p) v = v * x + c;
  return v;
}

// Real parts of all roots of p (highest degree first).  Degree <= 2 closed form (as
// Ceres), else Durand-Kerner.
void poly_roots_real(std::vector<double> p, std::vector<double>* real) {
  real->clear();
  size_t lead = 0;
  while (lead < p.size() && p[lead] == 0.0) ++lead;
  p.erase(p.begin(), p.begin() + lead);
  const int deg = static_cast<int>(p.size()) - 1;
  if (deg <= 0) return;
  if (deg == 1) { real->push_back(-p[1] / p[0]); return; }
  if (deg == 2) {
    const double a = p[0], b = p[1], c = p[2];
    const double D = b * b - 4 * a * c;
    const double sD = std::sqrt(std::fabs(D));
    if (D >= 0) {
      if (b >= 0) { real->push_back((-b - sD) / (2.0 * a)); real->push_back((2.0 * c) / (-b - sD)); }
      else { real->push_back((2.0 * c) / (-b + sD)); real->push_back((-b + sD) / (2.0 * a)); }
    } else { real->push_back(-b / (2.0 * a)); real->push_back(-b / (2.0 * a)); }
    return;
  }
  // Durand-Kerner, total-step form (every root is updated from the previous iterate of all roots), written out in
  // real arithmetic exactly as the CUDA kernel's warp-parallel version does it (one lane per root there).
  double c[8], zr[8], zi[8], qr[8], qi[8];
  for (int i = 0; i <= deg; ++i) c[i] = p[i] * (1.0 / p[0]);
  // Fujiwara's bound on the root moduli: 2 max_k |c_k|^(1/k) (the last coefficient halved)
  double radius = 0.0;
  for (int i = 1; i <= deg; ++i) {
    const double a = std::fabs(c[i]) * (i == deg ? 0.5 : 1.0);
    radius = std::max(radius, a > 0.0 ? std::exp(std::log(a) / (double)i) : 0.0);
  }
  radius = 2.0 * radius + 1e-300;
  for (int i = 0; i < deg; ++i) {
    const double ang = 2.0 * 3.14159265358979323846 * i / deg + 0.4;
    zr[i] = 0.5 * radius * std::cos(ang); zi[i] = 0.5 * radius * std::sin(ang);
  }
  for (int it = 0; it < 100; ++it) {
    double change = 0.0;
    for (int i = 0; i < deg; ++i) {
      double nr = 0.0, ni = 0.0;
      for (int k = 0; k <= deg; ++k) {
        const double tr = nr * zr[i] - ni * zi[i] + c[k];
        const double ti = nr * zi[i] + ni * zr[i];
        nr = tr; ni = ti;
      }
      double dr = 1.0, di = 0.0;
      for (int j = 0; j < deg; ++j) if (j != i) {
        const double er = zr[i] - zr[j], ei = zi[i] - zi[j];
        const double tr = dr * er - di * ei, ti = dr * ei + di * er;
        dr = tr; di = ti;
      }
      double den = dr * dr + di * di;
      if (den == 0.0) { dr = 1e-300; di = 0.0; den = dr * dr; if (den == 0.0) den = 1e-300; }
      const double iden = 1.0 / den;
      qr[i] = (nr * dr + ni * di) * iden; qi[i] = (ni * dr - nr * di) * iden;
      change = std::max(change, std::sqrt(qr[i] * qr[i] + qi[i] * qi[i]));
    }
    for (int i = 0; i < deg; ++i) { zr[i] -= qr[i]; zi[i] -= qi[i]; }
    if (change < 1e-14 * radius) break;
  }
  for (int i = 0; i < deg; ++i) real->push_back(zr[i]);
}

// Minimise the polynomial interpolating the samples over [xmin, xmax].
double interpolating_min_step(const Sample& lower, const Sample& previous, const Sample& current,
                              double xmin, double xmax) {
  if (!current.value_valid) return std::min(std::max(current.x * 0.5, xmin), xmax);
  // CUBIC interpolation (Ceres default line_search_interpolation_type).
  std::vector<Sample> s;
  s.push_back(lower);
  s.push_back(current);
  if (previous.value_valid) s.push_back(previous);
  int nc = 0;
  for (const Sample& q : s) { if (q.value_valid) ++nc; if (q.gradient_valid) ++nc; }
  const int deg = nc - 1;
  std::vector<double> M(nc * nc, 0.0), rhs(nc, 0.0);
  int row = 0;
  for (const Sample& q : s) {
    if (q.value_valid) {
      for (int j = 0; j <= deg; ++j) M[row * nc + j] = std::pow(q.x, deg - j);
      rhs[row] = q.value; ++row;
    }
    if (q.gradient_valid) {
      for (int j = 0; j < deg; ++j) M[row * nc + j] = (deg - j) * std::pow(q.x, deg - j - 1);
      rhs[row] = q.gradient; ++row;
    }
  }
  std::vector<double> poly(nc, 0.0);
  solve_full_pivot(nc, M, rhs, poly.data());
  double best_x = (xmin + xmax) / 2.0;
  double best_v = poly_eval(poly, best_x);
  const double vmin = poly_eval(poly, xmin);
  if (vmin < best_v) { best_v = vmin; best_x = xmin; }
  const double vmax = poly_eval(poly, xmax);
  if (vmax < best_v) { best_v = vmax; best_x = xmax; }
  if (poly.size() <= 2) return best_x;
  std::vector<double> der(poly.size() - 1);
  const int d = static_cast<int>(poly.size()) - 1;
  for (int j = 0; j < d; ++j) der[j] = (d - j) * poly[j];
  std::vector<double> roots;
  poly_roots_real(der, &roots);
  for (double root : roots) {
    if (root < xmin || root > xmax) continue;
    const double v = poly_eval(poly, root);
    if (v < best_v) { best_v = v; best_x = root; }
  }
  return best_x;
}

struct Stats {
  int32_t iterations;        // Ceres iteration index at termination
  int32_t successful_steps;
  int32_t unique_evals;      // distinct points a fused evaluator has to visit
  int32_t cost_evals;        // residual-only evaluations Ceres would perform
  int32_t jac_evals;         // residual+jacobian evaluations Ceres would perform
  int32_t line_search_steps; // Armijo contractions
  int32_t termination;       // 0 conv(grad) 1 conv(param) 2 conv(func) 3 no-conv(max iter) 4 conv(radius) 5 failure 6 infeasible
  int32_t reserved;
};

// ---------------------------------------------------------------------------
// Options of the parity tooling (all off = the reference behaviour restated above).
//   linear_solver 1: solve the damped normal equations (Js^T Js + D^2) y = Js^T r by Cholesky, with the model cost
//                    change from the same 4x4 / 6x6 quantities -- the arithmetic the CUDA kernel uses -- instead of
//                    Householder QR on the (m + P) x P stacked matrix (DENSE_QR, what Ceres does).
//   ext:             take cost, g = J^T r and J^T J of every evaluation from a callback (the CUDA evaluation kernel
//                    through tests/tools/trace_divergence.py) instead of the dual-number pass above: the oracle's
//                    CONTROL FLOW then runs on the kernel's sums, which separates control-logic differences from
//                    summation-order differences.  Needs linear_solver 1 (no Jacobian rows are available).
//   trace:           one 16-double record per evaluation, same layout as the kernel's frustum_solve_traced_f32.
// ---------------------------------------------------------------------------
typedef int (*ExternalEval)(void* user, const double* x6, double* cost, double* g6, double* JtJ36);
struct Options {
  int linear_solver = 0;
  ExternalEval ext = nullptr;
  void* ext_user = nullptr;
  double* trace = nullptr;
  int trace_cap = 0;
};
constexpr int kTraceRec = 16;

// Buffers reused across the iterations of one solve (no heap traffic inside the loop).
struct Workspace {
  Eval ev, trial;
  std::vector<double> Js, res, A, b;
};

// Cholesky solve of (As + diag(d2)) y = gs, As full symmetric P x P (the kernel's chol_solve, restated).
bool chol_solve(int P, const double As[6][6], const double* d2, const double* gs, double* y) {
  double L[6][6], inv[6], z[6];
  bool ok = true;
  for (int j = 0; j < P; ++j) {
    double sacc = As[j][j] + d2[j];
    for (int k = 0; k < j; ++k) sacc -= L[j][k] * L[j][k];
    if (!(sacc > 0.0)) ok = false;
    inv[j] = 1.0 / std::sqrt(sacc);
    L[j][j] = sacc * inv[j];
    for (int i = j + 1; i < P; ++i) {
      double t = As[i][j];
      for (int k = 0; k < j; ++k) t -= L[i][k] * L[j][k];
      L[i][j] = t * inv[j];
    }
  }
  for (int i = 0; i < P; ++i) {
    double t = gs[i];
    for (int k = 0; k < i; ++k) t -= L[i][k] * z[k];
    z[i] = t * inv[i];
  }
  for (int i = P - 1; i >= 0; --i) {
    double t = z[i];
    for (int k = i + 1; k < P; ++k) t -= L[k][i] * y[k];
    y[i] = t * inv[i];
  }
  return ok;
}

// ---------------------------------------------------------------------------
// The trust-region loop Ceres runs for the options at registration.cpp:137-147.
// ---------------------------------------------------------------------------
void minimize(const Problem& pb, double* x_user, int max_iter, Stats* st, const Options& opt, Workspace& wsp) {
  const int P = pb.P;
  std::memset(st, 0, sizeof(*st));
  const bool chol = opt.linear_solver == 1;
  const bool ext = opt.ext != nullptr;
  int n_rec = 0;
  double* rec = nullptr;
  auto trace_before = [&](const double* xt, double value, double x_cost, double radius, int iteration, int phase,
                          double alpha, double mcc) {
    rec = nullptr;
    if (opt.trace == nullptr || n_rec >= opt.trace_cap) { ++n_rec; return; }
    rec = opt.trace + (size_t)n_rec * kTraceRec;
    ++n_rec;
    for (int j = 0; j < 6; ++j) rec[j] = j < P ? xt[j] : 0.0;
    rec[6] = value; rec[7] = x_cost; rec[8] = radius; rec[9] = (double)iteration; rec[10] = (double)phase;
    rec[11] = 0.0; rec[12] = -1.0; rec[13] = alpha; rec[14] = mcc; rec[15] = 1.0;
  };
  auto trace_after = [&](int step_ok, int term) { if (rec) { rec[11] = (double)step_ok; rec[12] = (double)term; } };

  // Feasibility check (Program::IsFeasible) -- infeasible start => FAILURE, x untouched.
  for (int j = 0; j < P; ++j)
    if (x_user[j] < pb.lb[j] || x_user[j] > pb.ub[j]) { st->termination = 6; return; }

  double x[6], cand[6], delta[6], step[6], scale[6], diag[6];
  { double zero[6] = {0, 0, 0, 0, 0, 0}; plus_project(pb, x_user, zero, x); }
  double x_norm = 0.0; for (int j = 0; j < P; ++j) x_norm += x[j] * x[j]; x_norm = std::sqrt(x_norm);

  // One evaluation at xx: cost, gradient and (QR mode) corrected residuals / Jacobian rows or (Cholesky mode) J^T J.
  struct Sums { double cost, g[6], A[6][6]; };
  auto eval_at = [&](const double* xx, Eval* ev, Sums* sm) {
    if (ext) {
      double x6[6] = {0, 0, 0, 0, 0, 0}, g6[6], JtJ[36];
      for (int j = 0; j < P; ++j) x6[j] = xx[j];
      opt.ext(opt.ext_user, x6, &sm->cost, g6, JtJ);
      for (int j = 0; j < P; ++j) { sm->g[j] = g6[j]; for (int k = 0; k < P; ++k) sm->A[j][k] = JtJ[j * P + k]; }
      return;
    }
    evaluate(pb, xx, true, true, ev);
    sm->cost = ev->cost;
    for (int j = 0; j < P; ++j) sm->g[j] = ev->g[j];
    if (chol) {
      for (int j = 0; j < P; ++j) for (int k = j; k < P; ++k) {
        double acc = 0.0;
        for (int64_t i = 0; i < pb.rows; ++i) acc += ev->J[i * P + j] * ev->J[i * P + k];
        sm->A[j][k] = acc; sm->A[k][j] = acc;
      }
    }
  };

  Eval& ev = wsp.ev;
  Sums cur;                                 // sums at the current iterate x
  eval_at(x, &ev, &cur);
  st->jac_evals++; st->unique_evals++;
  double x_cost = cur.cost;
  const int64_t m = pb.rows;
  std::vector<double>& Js = wsp.Js;          // scaled in place below (QR mode)
  std::vector<double>& res = wsp.res;
  if (!chol) { Js = ev.J; res = ev.r; }
  double g[6]; for (int j = 0; j < P; ++j) g[j] = cur.g[j];

  // Jacobi scaling, computed once at iteration 0.
  for (int j = 0; j < P; ++j) {
    double s2 = 0.0;
    if (chol) s2 = cur.A[j][j];
    else for (int64_t i = 0; i < m; ++i) s2 += Js[i * P + j] * Js[i * P + j];
    scale[j] = 1.0 / (1.0 + std::sqrt(s2));
  }
  auto scale_columns = [&](std::vector<double>& Jm) {
    for (int64_t i = 0; i < m; ++i) for (int j = 0; j < P; ++j) Jm[i * P + j] *= scale[j];
  };
  if (!chol) scale_columns(Js);
  auto gradient_max_norm = [&](const double* xx, const double* gg) {
    double ng[6], proj[6], mx = 0.0;
    for (int j = 0; j < P; ++j) ng[j] = -gg[j];
    plus_project(pb, xx, ng, proj);
    for (int j = 0; j < P; ++j) mx = std::max(mx, std::fabs(xx[j] - proj[j]));
    return mx;
  };
  double grad_max = gradient_max_norm(x, g);

  double radius = 1e4, decrease_factor = 2.0;
  bool reuse_diag = false;
  bool step_successful = true;       // iteration 0 counts as successful
  int invalid = 0;
  int iteration = 0;
  double minimum_cost = x_cost;
  for (int j = 0; j < P; ++j) x_user[j] = x[j];
  st->successful_steps = 0;
  trace_before(x, x_cost, 0.0, radius, 0, 0, 1.0, 0.0);
  trace_after(1, -1);

  std::vector<double>& A = wsp.A;
  std::vector<double>& b = wsp.b;
  if (!chol) { A.resize((m + P) * P); b.resize(m + P); }
  Eval& trial = wsp.trial;           // evaluation at the current line-search sample
  Sums tsum;

  for (;;) {
    // --- loop-top termination tests (FinalizeIterationAndCheckIfMinimizerCanContinue)
    if (iteration >= max_iter) { st->termination = 3; break; }
    if (step_successful && grad_max <= 1e-10) { st->termination = 0; break; }
    if (radius <= 1e-32) { st->termination = 4; break; }
    ++iteration;
    step_successful = false;

    // --- LM step: min || [Js; sqrt(diag/radius)] y - [r; 0] ||  (DENSE_QR), step = -y
    double y[6];
    bool ok;
    double mcc = 0.0;
    if (chol) {
      double As[6][6], gs[6], d2[6];
      for (int j = 0; j < P; ++j) { gs[j] = g[j] * scale[j]; for (int k = 0; k < P; ++k) As[j][k] = cur.A[j][k] * scale[j] * scale[k]; }
      if (!reuse_diag) for (int j = 0; j < P; ++j) diag[j] = std::min(std::max(As[j][j], 1e-6), 1e32);
      reuse_diag = true;
      const double inv_radius = 1.0 / radius;
      for (int j = 0; j < P; ++j) d2[j] = diag[j] * inv_radius;
      ok = chol_solve(P, As, d2, gs, y);
      for (int j = 0; j < P; ++j) { step[j] = -y[j]; if (!std::isfinite(step[j])) ok = false; }
      if (ok) {
        double lin = 0.0, quad = 0.0;
        for (int j = 0; j < P; ++j) {
          lin += -y[j] * gs[j];
          double rowsum = 0.0;
          for (int k = 0; k < P; ++k) rowsum += As[j][k] * -y[k];
          quad += -y[j] * rowsum;
        }
        mcc = -lin - 0.5 * quad;
      }
    } else {
      if (!reuse_diag) {
        for (int j = 0; j < P; ++j) {
          double s2 = 0.0;
          for (int64_t i = 0; i < m; ++i) s2 += Js[i * P + j] * Js[i * P + j];
          diag[j] = std::min(std::max(s2, 1e-6), 1e32);
        }
      }
      reuse_diag = true;
      std::memcpy(A.data(), Js.data(), sizeof(double) * m * P);
      std::memset(A.data() + m * P, 0, sizeof(double) * P * P);
      for (int j = 0; j < P; ++j) A[(m + j) * P + j] = std::sqrt(diag[j] / radius);
      std::memcpy(b.data(), res.data(), sizeof(double) * m);
      std::memset(b.data() + m, 0, sizeof(double) * P);
      ok = householder_lstsq(A, b, m + P, P, y);
      for (int j = 0; j < P; ++j) { step[j] = -y[j]; if (!std::isfinite(step[j])) ok = false; }
      if (ok) {
        // model_cost_change = -(Js step)^T (r + Js step / 2)
        for (int64_t i = 0; i < m; ++i) {
          double mr = 0.0;
          for (int j = 0; j < P; ++j) mr += Js[i * P + j] * step[j];
          mcc -= mr * (res[i] + mr / 2.0);
        }
      }
    }
    if (!ok || !(mcc > 0.0)) {
      if (++invalid >= 5) { st->termination = 5; break; }
      // LevenbergMarquardtStrategy::StepIsInvalid() == StepRejected(0): radius /= decrease_factor, factor doubles
      radius = radius / decrease_factor; decrease_factor *= 2.0; reuse_diag = true;
      continue;
    }
    invalid = 0;
    for (int j = 0; j < P; ++j) delta[j] = step[j] * scale[j];

    // --- projected Armijo line search along delta (bounds-constrained problems)
    bool have_cand_eval = false;
    {
      double gd = 0.0, dmax = 0.0;
      for (int j = 0; j < P; ++j) { gd += g[j] * delta[j]; dmax = std::max(dmax, std::fabs(delta[j])); }
      Sample lower{0.0, x_cost, gd, true, true};
      Sample previous{0.0, 0.0, 0.0, false, false};
      Sample current{0.0, 0.0, 0.0, false, false};
      auto sample_at = [&](double alpha, Sample* s) {
        double sd[6], xt[6];
        for (int j = 0; j < P; ++j) sd[j] = alpha * delta[j];
        plus_project(pb, x, sd, xt);
        eval_at(xt, &trial, &tsum);
        st->jac_evals++; st->unique_evals++;
        s->x = alpha; s->value = tsum.cost; s->value_valid = std::isfinite(tsum.cost);
        double gr = 0.0; for (int j = 0; j < P; ++j) gr += delta[j] * tsum.g[j];
        s->gradient = gr; s->gradient_valid = s->value_valid && std::isfinite(gr);
        trace_before(xt, tsum.cost, x_cost, radius, iteration, 1, alpha, mcc);
      };
      sample_at(1.0, &current);
      int ls_iter = 0; bool success = true;
      while (!current.value_valid || current.value > x_cost + 1e-4 * gd * current.x) {
        ++ls_iter; st->line_search_steps++;
        if (ls_iter >= 20) { success = false; break; }
        const double a = interpolating_min_step(lower, previous, current, 1e-3 * current.x, 0.6 * current.x);
        if (a * dmax < 1e-9) { success = false; break; }
        previous = current;
        sample_at(a, &current);
      }
      if (success) {
        for (int j = 0; j < P; ++j) delta[j] *= current.x;
        have_cand_eval = true;      // candidate == last sample point, bit for bit
      }
    }

    // --- candidate point and its cost
    plus_project(pb, x, delta, cand);
    double cand_cost;
    if (have_cand_eval) { cand_cost = tsum.cost; st->cost_evals++; }
    else {
      eval_at(cand, &trial, &tsum); cand_cost = tsum.cost; st->cost_evals++; st->unique_evals++;
      trace_before(cand, cand_cost, x_cost, radius, iteration, 2, 1.0, mcc);
    }

    // --- parameter / function tolerance (x is NOT advanced when they fire)
    double sn = 0.0; for (int j = 0; j < P; ++j) sn += (x[j] - cand[j]) * (x[j] - cand[j]);
    if (std::sqrt(sn) <= 1e-8 * (x_norm + 1e-8)) { st->termination = 1; trace_after(0, 1); break; }
    if (std::fabs(x_cost - cand_cost) <= 1e-6 * x_cost) { st->termination = 2; trace_after(0, 2); break; }

    const double rho = (x_cost - cand_cost) / mcc;
    if (rho > 1e-3) {
      for (int j = 0; j < P; ++j) x[j] = cand[j];
      x_norm = 0.0; for (int j = 0; j < P; ++j) x_norm += x[j] * x[j]; x_norm = std::sqrt(x_norm);
      // Ceres re-evaluates residuals + Jacobian at the accepted point (same values).
      st->jac_evals++;
      x_cost = tsum.cost;
      cur = tsum;
      if (!chol) { Js.swap(trial.J); res.swap(trial.r); scale_columns(Js); }
      for (int j = 0; j < P; ++j) g[j] = tsum.g[j];
      grad_max = gradient_max_norm(x, g);
      radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * rho - 1.0, 3));
      radius = std::min(1e16, radius);
      decrease_factor = 2.0; reuse_diag = false;
      step_successful = true; st->successful_steps++;
      if (x_cost < minimum_cost) { minimum_cost = x_cost; for (int j = 0; j < P; ++j) x_user[j] = x[j]; }
      trace_after(1, -1);
    } else {
      radius = radius / decrease_factor; decrease_factor *= 2.0; reuse_diag = true;
      trace_after(0, -1);
    }
  }
  st->iterations = iteration;
  // the kernel's trace writes the termination code of loop-top exits into the last record
  if (opt.trace && n_rec > 0 && n_rec <= opt.trace_cap) {
    double* last = opt.trace + (size_t)(n_rec - 1) * kTraceRec;
    if (last[12] < 0.0) last[12] = (double)st->termination;
  }
}

// Pose matrix from the parameter vector (registration.cpp:161-185; AngleAxisToRotationMatrix).
void pose_from_params(const double* x, int P, double* P16) {
  double aa[3]; const double* t;
  if (P == 4) { aa[0] = 0; aa[1] = x[0]; aa[2] = 0; t = x + 1; } else { aa[0] = x[0]; aa[1] = x[1]; aa[2] = x[2]; t = x + 3; }
  double R[9];   // row-major R(i,j) = R[3 i + j]
  const double theta2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (theta2 > std::numeric_limits<double>::epsilon()) {
    const double theta = std::sqrt(theta2);
    const double wx = aa[0] / theta, wy = aa[1] / theta, wz = aa[2] / theta;
    const double c = std::cos(theta), s = std::sin(theta);
    R[0] = c + wx * wx * (1.0 - c);       R[3] = wz * s + wx * wy * (1.0 - c);  R[6] = -wy * s + wx * wz * (1.0 - c);
    R[1] = wx * wy * (1.0 - c) - wz * s;  R[4] = c + wy * wy * (1.0 - c);       R[7] = wx * s + wy * wz * (1.0 - c);
    R[2] = wy * s + wx * wz * (1.0 - c);  R[5] = -wx * s + wy * wz * (1.0 - c); R[8] = c + wz * wz * (1.0 - c);
  } else {
    R[0] = 1.0;    R[3] = aa[2];  R[6] = -aa[1];
    R[1] = -aa[2]; R[4] = 1.0;    R[7] = aa[0];
    R[2] = aa[1];  R[5] = -aa[0]; R[8] = 1.0;
  }
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) P16[4 * i + j] = R[3 * i + j]; P16[4 * i + 3] = t[i]; }
  P16[12] = 0; P16[13] = 0; P16[14] = 0; P16[15] = 1;
}

void setup_problem(Problem* pb, const double* pts, const int32_t* labels, int64_t n, const double* K9,
                   double H, double W, const double* lb3, const double* ub3, int is_2d) {
  pb->px = pts; pb->py = pts + n; pb->pz = pts + 2 * n;
  pb->label = labels; pb->n = n;
  pb->cam.fx = K9[0]; pb->cam.fy = K9[4]; pb->cam.cx = K9[2]; pb->cam.cy = K9[5];   // registration.cpp:79-82
  pb->cam.H1 = H - 1; pb->cam.W1 = W - 1;                                           // registration.cpp:21-22
  pb->P = is_2d ? 4 : 6; pb->toff = is_2d ? 1 : 3;
  for (int j = 0; j < 6; ++j) { pb->lb[j] = -std::numeric_limits<double>::max(); pb->ub[j] = std::numeric_limits<double>::max(); }
  for (int k = 0; k < 3; ++k) { pb->lb[pb->toff + k] = lb3[k]; pb->ub[pb->toff + k] = ub3[k]; }
  int64_t rows = 0;
  for (int64_t i = 0; i < n; ++i) rows += (labels[i] == 1) ? 3 : (labels[i] == 0 ? 1 : 0);
  pb->rows = rows;
}

}  // namespace

extern "C" {

// Number of residual rows n0 + 3 n1 for a label vector.
int64_t frustum_oracle_num_residuals(const int32_t* labels, int64_t n) {
  int64_t rows = 0;
  for (int64_t i = 0; i < n; ++i) rows += (labels[i] == 1) ? 3 : (labels[i] == 0 ? 1 : 0);
  return rows;
}

// Restatement of solvePGivenK (registration.cpp:9-186).  pts = [x[N] | y[N] | z[N]] f64.
// residuals may be NULL.  stats = 8 x int32 (struct Stats).  params_out = 6 doubles (final x).
// Parity-tooling extras (all 0 / NULL = the reference behaviour): linear_solver 1 = Cholesky on the normal equations;
// ext / ext_user = external evaluation callback (needs linear_solver 1); trace [trace_cap][16] per-evaluation records.
int frustum_oracle_solve_ex(const double* pts, const int32_t* labels, int64_t n, const double* K9,
                            double init_y_angle, const double* init_T, double H, double W,
                            const double* lb3, const double* ub3, int max_iter, int is_2d,
                            double* P16, double* final_cost, double* residuals, int32_t* stats,
                            double* params_out, int linear_solver, ExternalEval ext, void* ext_user,
                            double* trace, int trace_cap) {
  if (ext != nullptr && linear_solver != 1) return -1;
  Problem pb;
  setup_problem(&pb, pts, labels, n, K9, H, W, lb3, ub3, is_2d);
  double x[6] = {0, 0, 0, 0, 0, 0};
  if (is_2d) { x[0] = init_y_angle; for (int k = 0; k < 3; ++k) x[1 + k] = init_T[k]; }
  else { x[0] = 0; x[1] = init_y_angle; x[2] = 0; for (int k = 0; k < 3; ++k) x[3 + k] = init_T[k]; }
  Stats st;
  Options opt;
  opt.linear_solver = linear_solver; opt.ext = ext; opt.ext_user = ext_user; opt.trace = trace; opt.trace_cap = trace_cap;
  if (trace) std::memset(trace, 0, sizeof(double) * (size_t)trace_cap * kTraceRec);
  Workspace wsp;
  minimize(pb, x, max_iter, &st, opt, wsp);
  if (ext) {
    double g6[6], JtJ[36], x6[6] = {0, 0, 0, 0, 0, 0};
    for (int j = 0; j < pb.P; ++j) x6[j] = x[j];
    ext(ext_user, x6, final_cost, g6, JtJ);
  } else {
    evaluate(pb, x, false, residuals != nullptr, &wsp.ev);       // Problem::Evaluate, registration.cpp:150-155
    *final_cost = wsp.ev.cost;
    if (residuals) std::memcpy(residuals, wsp.ev.r.data(), sizeof(double) * pb.rows);
  }
  pose_from_params(x, pb.P, P16);
  if (stats) std::memcpy(stats, &st, sizeof(st));
  if (params_out) for (int j = 0; j < 6; ++j) params_out[j] = (j < pb.P) ? x[j] : 0.0;
  return 0;
}

int frustum_oracle_solve(const double* pts, const int32_t* labels, int64_t n, const double* K9,
                         double init_y_angle, const double* init_T, double H, double W,
                         const double* lb3, const double* ub3, int max_iter, int is_2d,
                         double* P16, double* final_cost, double* residuals, int32_t* stats,
                         double* params_out) {
  return frustum_oracle_solve_ex(pts, labels, n, K9, init_y_angle, init_T, H, W, lb3, ub3, max_iter, is_2d, P16,
                                 final_cost, residuals, stats, params_out, 0, nullptr, nullptr, nullptr, 0);
}

// One evaluation at an explicit parameter vector: cost, g = J^T r (P), JtJ (P x P row-major),
// optional corrected residual vector.  Used by tests to check the CUDA evaluation kernel.
int frustum_oracle_evaluate(const double* pts, const int32_t* labels, int64_t n, const double* K9,
                            const double* x, double H, double W, int is_2d,
                            double* cost, double* g, double* JtJ, double* residuals) {
  Problem pb;
  const double lb[3] = {-1e300, -1e300, -1e300}, ub[3] = {1e300, 1e300, 1e300};
  setup_problem(&pb, pts, labels, n, K9, H, W, lb, ub, is_2d);
  Eval ev;
  evaluate(pb, x, true, true, &ev);
  *cost = ev.cost;
  const int P = pb.P;
  for (int j = 0; j < P; ++j) g[j] = ev.g[j];
  for (int a = 0; a < P; ++a) for (int b = 0; b < P; ++b) {
    double s = 0.0;
    for (int64_t i = 0; i < pb.rows; ++i) s += ev.J[i * P + a] * ev.J[i * P + b];
    JtJ[a * P + b] = s;
  }
  if (residuals) std::memcpy(residuals, ev.r.data(), sizeof(double) * pb.rows);
  return 0;
}

}  // extern "C"
