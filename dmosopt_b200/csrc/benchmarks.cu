// Vectorised multi-objective benchmark functions (SURVEY.md section 8f row N4).
// The reference evaluates them one row at a time in Python (dmosopt/benchmarks/moo_benchmarks.py:21-497: DTLZ1-5, DTLZ7,
// WFG1, WFG4 and the many-objective MaF1, MaF2, MaF4; ZDT1 / ZDT3 are the example objectives,
// examples/example_dmosopt_zdt1.py:9-20, examples/example_dmosopt_zdt3.py:9-21), which becomes the bottleneck of every
// non-surrogate run (MOASMO.py:57-58, 107-108).  Here: one thread per row, float64, the reference's formulas term by term
// (sums in index order; results agree to ~1e-15 relative, NumPy sums pairwise).
#include <math_constants.h>

#include "common.cuh"

namespace {

constexpr int BM_MAXOBJ = 16;
constexpr double PI = 3.14159265358979323846;

enum {
  BM_ZDT1 = 0, BM_ZDT3 = 1, BM_DTLZ1 = 10, BM_DTLZ2 = 11, BM_DTLZ3 = 12, BM_DTLZ4 = 13, BM_DTLZ5 = 14, BM_DTLZ7 = 16,
  BM_WFG1 = 21, BM_WFG4 = 24, BM_MAF1 = 31, BM_MAF2 = 32, BM_MAF4 = 34
};

// MaF4's scale 10^(2i) (moo_benchmarks.py:495 multiplies by the Python int 10 ** (2 * i), i.e. its correctly rounded
// double): literals, because pow(10.0, e) need not round 10^24 and above (not exact in binary) correctly
__constant__ double BM_MAF4_SCALE[BM_MAXOBJ] = {1e0,  1e2,  1e4,  1e6,  1e8,  1e10, 1e12, 1e14,
                                                1e16, 1e18, 1e20, 1e22, 1e24, 1e26, 1e28, 1e30};

// f_i = scale * prod_{j < M-i-1} c(x_j) * (i > 0 ? s(x_{M-i-1}) : 1): the product form shared by DTLZ1-5 and the WFG shapes
template <class C, class S>
__device__ __forceinline__ void product_form(const double* v, int M, double scale, C c, S s, double* f) {
  for (int i = 0; i < M; ++i) {
    double fi = scale;
    for (int j = 0; j < M - i - 1; ++j) fi *= c(v[j]);
    if (i > 0) fi *= s(v[M - i - 1]);
    f[i] = fi;
  }
}

__global__ void benchmark_kernel(int problem, const double* __restrict__ X, int64_t n, int d, int M, double alpha,
                                 double* __restrict__ Y) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const double* x = X + r * d;
  double f[BM_MAXOBJ];
  const int k = d - M + 1;  // DTLZ: the last k variables drive g
  switch (problem) {
    case BM_ZDT1:
    case BM_ZDT3: {
      double s = 0.0;
      for (int j = 1; j < d; ++j) s += x[j];
      const double g = 1.0 + 9.0 / (d - 1) * s;
      f[0] = x[0];
      if (problem == BM_ZDT1)
        f[1] = g * (1.0 - sqrt(x[0] / g));
      else
        f[1] = g * (1.0 - sqrt(x[0] / g)) - (x[0] / g) * sin(10.0 * PI * x[0]);  // as the reference's example writes it (g h - j)
      break;
    }
    case BM_DTLZ1:
    case BM_DTLZ3:
    case BM_MAF1: {
      double s = 0.0;
      for (int j = d - k; j < d; ++j) {
        const double t = x[j] - 0.5;
        s += t * t - cos(20.0 * PI * t);
      }
      if (problem == BM_MAF1) {  // g is the bare sum (no 100 (k + ...)), and the scale 1 + g, not (1 + g) / 2
        product_form(x, M, 1.0 + s, [](double v) { return v; }, [](double v) { return 1.0 - v; }, f);
        break;
      }
      const double g = 100.0 * (k + s);
      if (problem == BM_DTLZ1)
        product_form(x, M, 0.5 * (1.0 + g), [](double v) { return v; }, [](double v) { return 1.0 - v; }, f);
      else
        product_form(x, M, 1.0 + g, [](double v) { return cos(v * PI / 2); }, [](double v) { return sin(v * PI / 2); }, f);
      break;
    }
    case BM_DTLZ2:
    case BM_DTLZ4:
    case BM_DTLZ5:
    case BM_MAF2:
    case BM_MAF4: {
      double g = 0.0;
      for (int j = d - k; j < d; ++j) {
        const double t = x[j] - 0.5;
        g += t * t;
      }
      if (problem == BM_DTLZ2 || problem == BM_MAF2 || problem == BM_MAF4) {  // MaF2 is DTLZ2's arithmetic
        product_form(x, M, 1.0 + g, [](double v) { return cos(v * PI / 2); }, [](double v) { return sin(v * PI / 2); }, f);
        if (problem == BM_MAF4)
          for (int i = 0; i < M; ++i) f[i] *= BM_MAF4_SCALE[i];
      } else if (problem == BM_DTLZ4) {
        product_form(x, M, 1.0 + g, [alpha](double v) { return cos(pow(v, alpha) * PI / 2); },
                     [alpha](double v) { return sin(pow(v, alpha) * PI / 2); }, f);
      } else {
        double th[BM_MAXOBJ];
        th[0] = x[0] * PI / 2;
        for (int i = 1; i < M - 1; ++i) th[i] = (1.0 + 2.0 * g * x[i]) / (2.0 * (1.0 + g)) * PI / 2;
        product_form(th, M, 1.0 + g, [](double v) { return cos(v); }, [](double v) { return sin(v); }, f);
      }
      break;
    }
    case BM_DTLZ7: {
      double s = 0.0;
      for (int j = d - k; j < d; ++j) s += x[j];
      const double g = 1.0 + 9.0 * (s / k);
      double h = 0.0;
      for (int i = 0; i < M - 1; ++i) {
        f[i] = x[i];
        h += f[i] / (1.0 + g) * (1.0 + sin(3.0 * PI * f[i]));
      }
      f[M - 1] = (1.0 + g) * ((double)M - h);
      break;
    }
    case BM_WFG1: {
      // y = x / (2 i); t2 = y on the first kk = M - 1 entries, 0.35 + 0.65 y^0.02 on the rest; shape vector = maxima over
      // ll = d - kk wide windows [i ll, (i + 1) ll) clipped at d, and the mean of the last ll entries
      const int kk = M - 1, ll = d - kk;
      auto t2 = [x, kk](int j) {
        const double y = x[j] / (2.0 * (j + 1));
        return j < kk ? y : 0.35 + 0.65 * pow(y, 0.02);
      };
      double xv[BM_MAXOBJ];
      for (int i = 0; i < M - 1; ++i) {
        const int lo = i * ll, hi = (i + 1) * ll < d ? (i + 1) * ll : d;
        double m = CUDART_NAN;  // empty window: refused on the host (np.max raises in the reference)
        if (lo < hi) {
          m = t2(lo);
          for (int j = lo + 1; j < hi && !isnan(m); ++j) {  // np.max propagates NaN, fmax would drop it
            const double v = t2(j);
            if (isnan(v) || v > m) m = v;
          }
        }
        xv[i] = m;
      }
      double s = 0.0;
      for (int j = d - ll; j < d; ++j) s += t2(j);
      xv[M - 1] = s / ll;
      product_form(xv, M, 1.0, [](double v) { return 1.0 - cos(v * PI / 2); }, [](double v) { return 1.0 - sin(v * PI / 2); }, f);
      for (int i = 0; i < M; ++i) f[i] *= (double)(i + 2);  // * (1 + arange(1, M + 1))
      break;
    }
    case BM_WFG4: {
      // y = x / (2 i); t1 = y + 0.35 - 0.15 cos(10 pi y - 5); shape vector = means over ll = d - (M - 1) wide windows
      const int kk = M - 1, ll = d - kk;
      double xv[BM_MAXOBJ];
      for (int i = 0; i < M; ++i) {
        const int lo = (i < M - 1) ? i * ll : d - ll;
        const int hi = (i < M - 1) ? ((i + 1) * ll < d ? (i + 1) * ll : d) : d;
        double s = 0.0;
        for (int j = lo; j < hi; ++j) {
          const double y = x[j] / (2.0 * (j + 1));
          s += y + 0.35 - 0.15 * cos(10.0 * PI * y - 5.0);
        }
        xv[i] = hi > lo ? s / (hi - lo) : CUDART_NAN;  // np.mean of an empty slice is nan in the reference as well
      }
      product_form(xv, M, 1.0, [](double v) { return 1.0 - cos(v * PI / 2); }, [](double v) { return 1.0 - sin(v * PI / 2); }, f);
      for (int i = 0; i < M; ++i) f[i] *= (double)(i + 2);  // * (1 + arange(1, M + 1))
      break;
    }
    default:
      for (int i = 0; i < M; ++i) f[i] = CUDART_NAN;
  }
  for (int i = 0; i < M; ++i) Y[r * M + i] = f[i];
}

}  // namespace

extern "C" {

int dmo_benchmark_eval(dmo_ctx* ctx, int problem, const double* X, int64_t n, int n_var, int n_obj, double alpha, double* Y) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  if (n == 0) return DMO_OK;
  DMO_REQUIRE(n > 0 && X && Y && n_var >= 2 && n_obj >= 2 && n_obj <= BM_MAXOBJ, "benchmark_eval: bad arguments");
  const bool zdt = problem == BM_ZDT1 || problem == BM_ZDT3;
  const bool known = zdt || problem == BM_DTLZ1 || problem == BM_DTLZ2 || problem == BM_DTLZ3 || problem == BM_DTLZ4 ||
                     problem == BM_DTLZ5 || problem == BM_DTLZ7 || problem == BM_WFG1 || problem == BM_WFG4 ||
                     problem == BM_MAF1 || problem == BM_MAF2 || problem == BM_MAF4;
  if (!known) return dmo_fail(ctx, DMO_ERR_UNSUPPORTED, "benchmark_eval: unknown problem id %d", problem);
  DMO_REQUIRE(!zdt || n_obj == 2, "benchmark_eval: ZDT problems have two objectives");
  DMO_REQUIRE(zdt || n_var >= n_obj, "benchmark_eval: n_var must be at least n_obj");
  // WFG1's maximum windows start at i (n_var - n_obj + 1), i < n_obj - 1; where the last start reaches n_var, that
  // window is empty and the reference's np.max raises
  DMO_REQUIRE(problem != BM_WFG1 || (int64_t)(n_obj - 2) * (n_var - n_obj + 1) < n_var,
              "benchmark_eval: WFG1 with n_obj %d, n_var %d has an empty shape window ((n_obj - 2) (n_var - n_obj + 1) >= n_var)",
              n_obj, n_var);
  In<double> x;
  Out<double> y;
  DMO_TRY(x.init(ctx, X, (size_t)n * n_var));
  DMO_TRY(y.init(ctx, Y, (size_t)n * n_obj));
  DMO_LAUNCH(benchmark_kernel, (unsigned)ceil_div(n, 128), 128, 0, problem, x.d, n, n_var, n_obj, alpha, y.d);
  DMO_CHECK_LAUNCH();
  DMO_TRY(y.finish(ctx));
  DMO_CUDA(dmo_wait(ctx));
  return DMO_OK;
}

}  // extern "C"
