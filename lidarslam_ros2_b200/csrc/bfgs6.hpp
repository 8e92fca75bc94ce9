// BFGS driver of the GICP engine (product code; the oracle keeps its own copy under oracle/).
// Implements the minimiser the reference calls at gicp_omp_impl.hpp:209-230 — PCL 1.12 `BFGS<Functor>`
// (pcl/registration/bfgs.h, external), a port of GSL's vector_bfgs2 + Fletcher bracketing/sectioning line search
// (multimin/linear_minimize.c) — with sigma=0.01, rho=0.01, tau1=9, tau2=0.05, tau3=0.5, order=3.
// The 6-vector state machine is __host__ __device__ and templated on the functor. The engine instantiates it inside the
// persistent inner-loop kernel (gicp.cu: every thread of the controller CTA executes it redundantly and identically, so
// that the whole CTA takes part in each functor evaluation); tests/hostmath compiles it with g++ to compare it with the
// oracle's BFGS.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define B200_BFGS_HD __host__ __device__
#else
#define B200_BFGS_HD
#endif

namespace b200 {

constexpr double BFGS_DBL_EPSILON = 2.220446049250313e-16;

enum BfgsStatus { BFGS_NegativeGradientEpsilon = -3, BFGS_NotStarted = -2, BFGS_Running = -1, BFGS_Success = 0, BFGS_NoProgress = 1 };

template <class Functor>
class Bfgs6T {
 public:
  static constexpr int N = 6;
  struct Parameters {
    int bracket_iters = 100, section_iters = 100;
    double rho = 0.01, sigma = 0.01, tau1 = 9, tau2 = 0.05, tau3 = 0.5, step_size = 1;
    int order = 3;
  } parameters;
  double f = 0;
  double gradient[N];
  int n_f = 0, n_df = 0, n_fdf = 0;  // instrumentation

  B200_BFGS_HD explicit Bfgs6T(Functor& fn) : functor(fn) {}

  B200_BFGS_HD BfgsStatus minimizeInit(double* x) {
    delta_f = 0;
    for (int i = 0; i < N; i++) dx[i] = 0;
    functor.fdf(x, f, gradient);
    n_fdf++;
    copy(x0, x);
    copy(g0, gradient);
    g0norm = norm(g0);
    for (int i = 0; i < N; i++) p[i] = gradient[i] * -1 / g0norm;
    pnorm = norm(p);
    fp0 = -g0norm;
    changeDirection();
    return BFGS_NotStarted;
  }

  B200_BFGS_HD BfgsStatus minimizeOneStep(double* x) {
    double alpha = 0.0, alpha1;
    double f0 = f;
    if (pnorm == 0.0 || g0norm == 0.0 || fp0 == 0) {
      for (int i = 0; i < N; i++) dx[i] = 0;
      return BFGS_NoProgress;
    }
    if (delta_f < 0) {
      double del = fmax(-delta_f, 10 * BFGS_DBL_EPSILON * fabs(f0));
      alpha1 = fmin(1.0, 2.0 * del / (-fp0));
    } else {
      alpha1 = fabs(parameters.step_size);
    }
    BfgsStatus status = lineSearch(parameters.rho, parameters.sigma, parameters.tau1, parameters.tau2,
                                   parameters.tau3, parameters.order, alpha1, alpha);
    if (status != BFGS_Success) return status;
    updatePosition(alpha, x);
    delta_f = f - f0;
    {
      double dx0[N], dg0[N];
      for (int i = 0; i < N; i++) {
        dx0[i] = x[i] - x0[i];
        dx[i] = dx0[i];
        dg0[i] = gradient[i] - g0[i];
      }
      double dxg = dot(dx0, gradient), dgg = dot(dg0, gradient), dxdg = dot(dx0, dg0), dgnorm = norm(dg0);
      double A, B;
      if (dxdg != 0) {
        B = dxg / dxdg;
        A = -(1.0 + dgnorm * dgnorm / dxdg) * B + dgg / dxdg;
      } else {
        B = 0;
        A = 0;
      }
      for (int i = 0; i < N; i++) p[i] = -A * dx0[i] + gradient[i] - B * dg0[i];
    }
    copy(g0, gradient);
    copy(x0, x);
    g0norm = norm(g0);
    pnorm = norm(p);
    double dir = (dot(p, gradient) > 0) ? -1.0 : 1.0;
    for (int i = 0; i < N; i++) p[i] *= dir / pnorm;
    pnorm = norm(p);
    fp0 = dot(p, g0);
    changeDirection();
    return BFGS_Success;
  }

  // pre-1.11 PCL semantic `testGradient(epsilon)`: Success iff |g| < epsilon (see gicp.hpp header note)
  B200_BFGS_HD BfgsStatus testGradient(double epsilon) const {
    if (epsilon < 0) return BFGS_NegativeGradientEpsilon;
    return norm(gradient) < epsilon ? BFGS_Success : BFGS_Running;
  }

 private:
  Functor& functor;
  double delta_f = 0, fp0 = 0, pnorm = 0, g0norm = 0;
  double x0[N], g0[N], dx[N], p[N];
  double f_alpha = 0, df_alpha = 0, x_alpha[N], g_alpha[N];
  double f_cache_key = 0, df_cache_key = 0, x_cache_key = 0, g_cache_key = 0;

  B200_BFGS_HD static void copy(double* d, const double* s) { for (int i = 0; i < N; i++) d[i] = s[i]; }
  B200_BFGS_HD static double dot(const double* a, const double* b) { double s = 0; for (int i = 0; i < N; i++) s += a[i] * b[i]; return s; }
  B200_BFGS_HD static double norm(const double* a) { return sqrt(dot(a, a)); }

  B200_BFGS_HD void changeDirection() {
    copy(x_alpha, x0);
    x_cache_key = 0;
    f_alpha = f;
    f_cache_key = 0;
    copy(g_alpha, g0);
    g_cache_key = 0;
    df_alpha = slope();
    df_cache_key = 0;
  }
  B200_BFGS_HD void moveTo(double alpha) {
    if (alpha == x_cache_key) return;
    for (int i = 0; i < N; i++) x_alpha[i] = x0[i] + alpha * p[i];
    x_cache_key = alpha;
  }
  B200_BFGS_HD double slope() const { return dot(g_alpha, p); }
  B200_BFGS_HD double applyF(double alpha) {
    if (alpha == f_cache_key) return f_alpha;
    moveTo(alpha);
    f_alpha = functor.f(x_alpha);
    n_f++;
    f_cache_key = alpha;
    return f_alpha;
  }
  B200_BFGS_HD double applyDF(double alpha) {
    if (alpha == df_cache_key) return df_alpha;
    moveTo(alpha);
    if (alpha != g_cache_key) {
      functor.df(x_alpha, g_alpha);
      n_df++;
      g_cache_key = alpha;
    }
    df_alpha = slope();
    df_cache_key = alpha;
    return df_alpha;
  }
  B200_BFGS_HD void applyFDF(double alpha, double& fo, double& dfo) {
    if (alpha == f_cache_key && alpha == df_cache_key) {
      fo = f_alpha;
      dfo = df_alpha;
      return;
    }
    if (alpha == f_cache_key || alpha == df_cache_key) {
      fo = applyF(alpha);
      dfo = applyDF(alpha);
      return;
    }
    moveTo(alpha);
    functor.fdf(x_alpha, f_alpha, g_alpha);
    n_fdf++;
    f_cache_key = alpha;
    g_cache_key = alpha;
    df_alpha = slope();
    df_cache_key = alpha;
    fo = f_alpha;
    dfo = df_alpha;
  }
  B200_BFGS_HD void updatePosition(double alpha, double* x) {
    double fa, dfa;
    applyFDF(alpha, fa, dfa);
    f = f_alpha;
    copy(x, x_alpha);
    copy(gradient, g_alpha);
  }

  B200_BFGS_HD static double cubic(double c0, double c1, double c2, double c3, double z) { return c0 + z * (c1 + z * (c2 + z * c3)); }
  B200_BFGS_HD static void check_extremum(double c0, double c1, double c2, double c3, double z, double& zmin, double& fmin) {
    double y = cubic(c0, c1, c2, c3, z);
    if (y < fmin) {
      zmin = z;
      fmin = y;
    }
  }
  B200_BFGS_HD static int solve_quadratic(double a, double b, double c, double& x0, double& x1) {
    if (a == 0) {
      if (b == 0) return 0;
      x0 = -c / b;
      return 1;
    }
    double disc = b * b - 4 * a * c;
    if (disc > 0) {
      if (b == 0) {
        double r = sqrt(-c / a);
        x0 = -r;
        x1 = r;
      } else {
        double sgnb = (b > 0 ? 1 : -1);
        double temp = -0.5 * (b + sgnb * sqrt(disc));
        double r1 = temp / a, r2 = c / temp;
        if (r1 < r2) { x0 = r1; x1 = r2; } else { x0 = r2; x1 = r1; }
      }
      return 2;
    } else if (disc == 0) {
      x0 = -0.5 * b / a;
      x1 = -0.5 * b / a;
      return 2;
    }
    return 0;
  }
  B200_BFGS_HD static double interp_quad(double f0, double fp0, double f1, double zl, double zh, double& zmin_out) {
    double fl = f0 + zl * (fp0 + zl * (f1 - f0 - fp0));
    double fh = f0 + zh * (fp0 + zh * (f1 - f0 - fp0));
    double c = 2 * (f1 - f0 - fp0);
    double zmin = zl, fmin = fl;
    if (fh < fmin) { zmin = zh; fmin = fh; }
    if (c > 0) {
      double z = -fp0 / c;
      if (z > zl && z < zh) {
        double fz = f0 + z * (fp0 + z * (f1 - f0 - fp0));
        if (fz < fmin) { zmin = z; fmin = fz; }
      }
    }
    zmin_out = zmin;
    return fmin;
  }
  B200_BFGS_HD static double interp_cubic(double f0, double fp0, double f1, double fp1, double zl, double zh, double& zmin_out) {
    double eta = 3 * (f1 - f0) - 2 * fp0 - fp1;
    double xi = fp0 + fp1 - 2 * (f1 - f0);
    double c0 = f0, c1 = fp0, c2 = eta, c3 = xi;
    double zmin = zl, fmin = cubic(c0, c1, c2, c3, zl);
    check_extremum(c0, c1, c2, c3, zh, zmin, fmin);
    double z0 = 0, z1 = 0;
    int n = solve_quadratic(3 * c3, 2 * c2, c1, z0, z1);
    if (n == 2) {
      if (z0 > zl && z0 < zh) check_extremum(c0, c1, c2, c3, z0, zmin, fmin);
      if (z1 > zl && z1 < zh) check_extremum(c0, c1, c2, c3, z1, zmin, fmin);
    } else if (n == 1) {
      if (z0 > zl && z0 < zh) check_extremum(c0, c1, c2, c3, z0, zmin, fmin);
    }
    zmin_out = zmin;
    return fmin;
  }
  B200_BFGS_HD static double interpolate(double a, double fa, double fpa, double b, double fb, double fpb, double xmin, double xmax,
                            int order) {
    double y, ymin = (xmin - a) / (b - a), ymax = (xmax - a) / (b - a);
    if (ymin > ymax) {
      const double t = ymin;
      ymin = ymax;
      ymax = t;
    }
    if (order > 2 && (fpb == fpb)) interp_cubic(fa, fpa * (b - a), fb, fpb * (b - a), ymin, ymax, y);
    else interp_quad(fa, fpa * (b - a), fb, ymin, ymax, y);
    return a + y * (b - a);
  }

  B200_BFGS_HD BfgsStatus lineSearch(double rho, double sigma, double tau1, double tau2, double tau3, int order, double alpha1,
                        double& alpha_new) {
    double f0, fp0l, falpha, falpha_prev, fpalpha = 0, fpalpha_prev, delta, alpha_next;
    double alpha = alpha1, alpha_prev = 0.0;
    double a, b, fa, fb, fpa, fpb;
    int i = 0;
    applyFDF(0.0, f0, fp0l);
    falpha_prev = f0;
    fpalpha_prev = fp0l;
    a = 0.0; b = alpha;
    fa = f0; fb = 0.0;
    fpa = fp0l; fpb = 0.0;
    while (i++ < parameters.bracket_iters) {
      falpha = applyF(alpha);
      if (falpha > f0 + alpha * rho * fp0l || falpha >= falpha_prev) {
        a = alpha_prev; fa = falpha_prev; fpa = fpalpha_prev;
        b = alpha; fb = falpha; fpb = nan("");
        break;
      }
      fpalpha = applyDF(alpha);
      if (fabs(fpalpha) <= -sigma * fp0l) {
        alpha_new = alpha;
        return BFGS_Success;
      }
      if (fpalpha >= 0) {
        a = alpha; fa = falpha; fpa = fpalpha;
        b = alpha_prev; fb = falpha_prev; fpb = fpalpha_prev;
        break;
      }
      delta = alpha - alpha_prev;
      {
        double lower = alpha + delta, upper = alpha + tau1 * delta;
        alpha_next = interpolate(alpha_prev, falpha_prev, fpalpha_prev, alpha, falpha, fpalpha, lower, upper, order);
      }
      alpha_prev = alpha;
      falpha_prev = falpha;
      fpalpha_prev = fpalpha;
      alpha = alpha_next;
    }
    while (i++ < parameters.section_iters) {
      delta = b - a;
      {
        double lower = a + tau2 * delta, upper = b - tau3 * delta;
        alpha = interpolate(a, fa, fpa, b, fb, fpb, lower, upper, order);
      }
      falpha = applyF(alpha);
      if ((a - alpha) * fpa <= BFGS_DBL_EPSILON) return BFGS_NoProgress;
      if (falpha > f0 + rho * alpha * fp0l || falpha >= fa) {
        b = alpha; fb = falpha; fpb = nan("");
      } else {
        fpalpha = applyDF(alpha);
        if (fabs(fpalpha) <= -sigma * fp0l) {
          alpha_new = alpha;
          return BFGS_Success;
        }
        if (((b - a) >= 0 && fpalpha >= 0) || ((b - a) <= 0 && fpalpha <= 0)) {
          b = a; fb = fa; fpb = fpa;
          a = alpha; fa = falpha; fpa = fpalpha;
        } else {
          a = alpha; fa = falpha; fpa = fpalpha;
        }
      }
    }
    return BFGS_Success;
  }
};

}  // namespace b200
