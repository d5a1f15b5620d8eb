// Gaussian-process scoring of a hyper-parameter search round (il_b200/hpo.py): the posterior of M candidates under a zero-mean GP with a
// Matérn-5/2 ARD kernel, and q greedy expected-improvement picks with the kriging believer. The GP is fitted on the host (torch, fp64); these
// kernels take its Cholesky factor and weights. All arithmetic is fp64 on the CUDA cores (DFMA); every sum runs in an order fixed by the
// sizes, so results repeat bit for bit.
#include "common.cuh"

namespace {

constexpr int POST_THREADS = 256;  // one candidate per thread; __launch_bounds__(POST_THREADS, 2) keeps two blocks per SM (<= 128 registers)
constexpr int TB = 32;             // rows of the blocked forward substitution: a thread keeps TB partial sums in registers
constexpr int SEL_THREADS = 256;
constexpr int RED_THREADS = 1024;

struct GpHyper {
  double inv_ls[IL_GP_MAX_D];  // 1 / lengthscale per dimension
  double s2;                   // output scale (prior variance)
  double noise;                // Gaussian noise variance sigma_n^2 (jitter included)
};

// k(r^2) of the Matérn-5/2 kernel on a squared scaled distance: s2 (1 + sqrt5 r + 5 r^2 / 3) exp(-sqrt5 r)
__device__ __forceinline__ double matern52(double r2, double s2) {
  const double r = sqrt(r2);
  const double sr = 2.23606797749978969641 * r;
  return s2 * (1.0 + sr + (5.0 / 3.0) * r2) * exp(-sr);
}

// Posterior of candidate m (one thread each): rows [i0, i0 + TB) of k* = k(x_m, X) are formed on the fly from X (staged in shared memory,
// scaled by 1 / lengthscale) and the candidate's column of Ct, then reduced against the finished rows of V = L^-1 K*^T block by block (the
// TB x TB tile of L in shared memory, read as a broadcast), then solved against the diagonal tile. mu = k* . alpha accumulates on the way,
// and var = s2 - |v|^2 at the end. V [n (+ more), M] is written row by row, so a warp's loads and stores of one row are coalesced.
__global__ void __launch_bounds__(POST_THREADS, 2) gp_posterior_kernel(const double* __restrict__ X, const double* __restrict__ alpha, const double* __restrict__ L, int n, int d,
                                                                     const double* __restrict__ Ct, int64_t M, GpHyper hp, double* __restrict__ mu, double* __restrict__ var,
                                                                     double* __restrict__ V) {
  __shared__ double xs[TB][IL_GP_MAX_D + 1];
  __shared__ double2 lt2[TB][TB / 2];  // double2 storage: 16-byte aligned for the paired reads below
  double(*lt)[TB] = reinterpret_cast<double(*)[TB]>(lt2);  // lt[j][i] = L[i0 + i][j0 + j]: for one j, consecutive i are consecutive words
  const int64_t m = (int64_t)blockIdx.x * POST_THREADS + threadIdx.x;
  const bool live = m < M;
  const int64_t mc = live ? m : M - 1;
  double mean = 0.0, vv = 0.0;
  for (int i0 = 0; i0 < n; i0 += TB) {
    const int rows = min(TB, n - i0);
    __syncthreads();
    for (int e = threadIdx.x; e < TB * d; e += POST_THREADS) {
      const int i = e / d, k = e % d;
      xs[i][k] = i < rows ? X[(int64_t)(i0 + i) * d + k] * hp.inv_ls[k] : 0.0;
    }
    __syncthreads();
    double acc[TB];
#pragma unroll
    for (int i = 0; i < TB; ++i) acc[i] = 0.0;
    for (int k = 0; k < d; ++k) {
      const double c = Ct[(int64_t)k * M + mc] * hp.inv_ls[k];
#pragma unroll
      for (int i = 0; i < TB; ++i) {
        const double t = c - xs[i][k];
        acc[i] = fma(t, t, acc[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      acc[i] = i < rows ? matern52(acc[i], hp.s2) : 0.0;
      if (i < rows) mean = fma(acc[i], alpha[i0 + i], mean);
    }
    for (int j0 = 0; j0 <= i0; j0 += TB) {  // the off-diagonal tiles, then the diagonal one
      __syncthreads();
      for (int e = threadIdx.x; e < TB * TB; e += POST_THREADS) {
        const int j = e / TB, i = e % TB;
        const bool in = i < rows && j0 + j < n;
        lt[j][i] = in ? L[(int64_t)(i0 + i) * n + j0 + j] : (j0 == i0 && i == j ? 1.0 : 0.0);
      }
      __syncthreads();
      if (j0 < i0) {
        for (int j = 0; j < TB; ++j) {
          const double vj = V[(int64_t)(j0 + j) * M + mc];
#pragma unroll
          for (int i = 0; i < TB; i += 2) {
            const double2 l2 = lt2[j][i / 2];
            acc[i] = fma(-l2.x, vj, acc[i]);
            acc[i + 1] = fma(-l2.y, vj, acc[i + 1]);
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < TB; ++j) {
          const double vj = acc[j] / lt[j][j];
          acc[j] = vj;
#pragma unroll
          for (int i = j + 1; i < TB; ++i) acc[i] = fma(-lt[j][i], vj, acc[i]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      if (i < rows) {
        vv = fma(acc[i], acc[i], vv);
        if (live) V[(int64_t)(i0 + i) * M + m] = acc[i];
      }
    }
  }
  if (live) {
    mu[m] = mean;
    var[m] = hp.s2 - vv;
  }
}

// ---- greedy batch selection ----------------------------------------------------------------------------------------------------
// Device state of one il_gp_select call, in its workspace.
struct SelState {
  double fstar;   // best believed value so far
  double s2w;     // var(x_w) before the current pick's update
  int count;      // admitted groups
  int done;       // no admissible candidate was left: later picks are -1
};

__device__ __forceinline__ double expected_improvement(double mu, double var, double fstar) {
  const double s = sqrt(fmax(var, 0.0));
  const double imp = mu - fstar;
  if (!(s > 0.0)) return fmax(imp, 0.0);
  const double z = imp / s;
  return imp * normcdf(z) + s * (0.3989422804014326779399 * exp(-0.5 * z * z));
}

// (value, index) argmax: the larger value wins, the smaller index on a tie; masked candidates carry -inf and index -1 never wins
__device__ __forceinline__ void arg_better(double& v, int64_t& i, double v2, int64_t i2) {
  if (i2 >= 0 && (i < 0 || v2 > v || (v2 == v && i2 < i))) v = v2, i = i2;
}

__device__ void block_argmax(double v, int64_t i, double* sv, int64_t* si, double* out_v, int64_t* out_i) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double v2 = __shfl_down_sync(0xffffffffu, v, o);
    const int64_t i2 = __shfl_down_sync(0xffffffffu, i, o);
    arg_better(v, i, v2, i2);
  }
  if (lane == 0) sv[warp] = v, si[warp] = i;
  __syncthreads();
  if (threadIdx.x == 0) {
    double bv = sv[0];
    int64_t bi = si[0];
    for (int w = 1; w < nw; ++w) arg_better(bv, bi, sv[w], si[w]);
    *out_v = bv, *out_i = bi;
  }
}

// Whether candidate m may still be picked: not picked yet, and (with max_groups G > 0) its group is admitted or fewer than G groups are.
__device__ __forceinline__ bool admissible(int64_t m, const int32_t* picked, const int32_t* group, int G, const int32_t* admitted, int count) {
  if (picked[m]) return false;
  if (G <= 0 || count < G) return true;
  const int g = group[m];
  for (int a = 0; a < count; ++a)
    if (admitted[a] == g) return true;
  return false;
}

// The streaming pass of pick j (w = the pick, r = n + j its row of V), then each block's argmax of the next pick's EI. With w < 0 (the first
// launch) only the EI partials are formed, from the posterior as il_gp_posterior left it.
__global__ void __launch_bounds__(SEL_THREADS) gp_select_pass_kernel(int64_t M, int d, int r, GpHyper hp, const double* __restrict__ Ct, const double* __restrict__ mu,
                                                                     double* __restrict__ var, double* __restrict__ V, const int32_t* __restrict__ group, int G,
                                                                     const int32_t* __restrict__ picked, const int32_t* __restrict__ admitted, const SelState* __restrict__ st,
                                                                     const double* __restrict__ vw, const double* __restrict__ xw, int first, double* __restrict__ part_v,
                                                                     int64_t* __restrict__ part_i) {
  __shared__ double sv[SEL_THREADS / 32];
  __shared__ int64_t si[SEL_THREADS / 32];
  const int64_t m = (int64_t)blockIdx.x * SEL_THREADS + threadIdx.x;
  double best = -INFINITY;
  int64_t bi = -1;
  if (!st->done && m < M) {
    double s2 = var[m];
    if (!first) {
      double r2 = 0.0;
      for (int k = 0; k < d; ++k) {
        const double t = (Ct[(int64_t)k * M + m] - xw[k]) * hp.inv_ls[k];
        r2 = fma(t, t, r2);
      }
      double c0 = 0.0, c1 = 0.0, c2 = 0.0, c3 = 0.0;  // v(x) . v(x_w), four chains in a fixed order
      int i = 0;
      for (; i + 4 <= r; i += 4) {
        c0 = fma(V[(int64_t)i * M + m], vw[i], c0);
        c1 = fma(V[(int64_t)(i + 1) * M + m], vw[i + 1], c1);
        c2 = fma(V[(int64_t)(i + 2) * M + m], vw[i + 2], c2);
        c3 = fma(V[(int64_t)(i + 3) * M + m], vw[i + 3], c3);
      }
      for (; i < r; ++i) c0 = fma(V[(int64_t)i * M + m], vw[i], c0);
      const double c = matern52(r2, hp.s2) - ((c0 + c1) + (c2 + c3));
      const double den = st->s2w + hp.noise;
      s2 -= c * c / den;
      var[m] = s2;
      V[(int64_t)r * M + m] = c / sqrt(den);
    }
    if (admissible(m, picked, group, G, admitted, st->count)) best = expected_improvement(mu[m], s2, st->fstar), bi = m;
  }
  block_argmax(best, bi, sv, si, part_v + blockIdx.x, part_i + blockIdx.x);
}

// One block: the argmax over the pass's block partials is pick j; record it, admit its group, snapshot var(x_w), raise f*, and gather
// v(x_w) (rows [0, n + j) of V's column w) and x_w for the next pass.
__global__ void __launch_bounds__(RED_THREADS) gp_select_pick_kernel(int nb, int64_t M, int d, int rows, const double* __restrict__ part_v, const int64_t* __restrict__ part_i,
                                                                     const double* __restrict__ Ct, const double* __restrict__ mu, const double* __restrict__ var,
                                                                     const double* __restrict__ V, const int32_t* __restrict__ group, int G, int32_t* __restrict__ picked,
                                                                     int32_t* __restrict__ admitted, SelState* __restrict__ st, double* __restrict__ vw, double* __restrict__ xw,
                                                                     int j, int32_t* __restrict__ picks, double* __restrict__ ei) {
  __shared__ double sv[RED_THREADS / 32];
  __shared__ int64_t si[RED_THREADS / 32];
  __shared__ double bv;
  __shared__ int64_t bi;
  double v = -INFINITY;
  int64_t i = -1;
  for (int b = threadIdx.x; b < nb; b += RED_THREADS) arg_better(v, i, part_v[b], part_i[b]);
  block_argmax(v, i, sv, si, &bv, &bi);
  __syncthreads();
  const int64_t w = st->done ? -1 : bi;
  __syncthreads();  // every thread has read st->done before thread 0 may set it
  if (w < 0) {
    if (threadIdx.x == 0) {
      picks[j] = -1;
      ei[j] = NAN;
      st->done = 1;
    }
    return;
  }
  if (threadIdx.x == 0) {
    picks[j] = (int32_t)w;
    ei[j] = bv;
    picked[w] = 1;
    if (G > 0) {
      bool seen = false;
      for (int a = 0; a < st->count; ++a) seen |= admitted[a] == group[w];
      if (!seen) admitted[st->count++] = group[w];
    }
    st->s2w = var[w];
    st->fstar = fmax(st->fstar, mu[w]);
  }
  for (int k = threadIdx.x; k < rows; k += RED_THREADS) vw[k] = V[(int64_t)k * M + w];
  for (int k = threadIdx.x; k < d; k += RED_THREADS) xw[k] = Ct[(int64_t)k * M + w];
}

__global__ void gp_select_init_kernel(int64_t M, double fstar, int32_t* __restrict__ picked, SelState* __restrict__ st) {
  const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m < M) picked[m] = 0;
  if (m == 0) *st = SelState{fstar, 0.0, 0, 0};
}

struct SelLayout {
  int64_t picked, admitted, state, vw, xw, part_v, part_i, total;
};

SelLayout sel_layout(int n, int d, int64_t M, int q) {
  const int64_t nb = (M + SEL_THREADS - 1) / SEL_THREADS;
  SelLayout s;
  int64_t off = 0;
  auto take = [&](int64_t bytes) { const int64_t o = off; off = il_align_up(off + bytes, 256); return o; };
  s.picked = take(M * (int64_t)sizeof(int32_t));
  s.admitted = take((int64_t)q * sizeof(int32_t));
  s.state = take(sizeof(SelState));
  s.vw = take((int64_t)(n + q) * sizeof(double));
  s.xw = take((int64_t)d * sizeof(double));
  s.part_v = take(nb * (int64_t)sizeof(double));
  s.part_i = take(nb * (int64_t)sizeof(int64_t));
  s.total = off;
  return s;
}

int make_hyper(const double* lengthscales, int d, double outputscale, double noise, GpHyper* hp, const char* who) {
  IL_CHECK(lengthscales, "%s: null pointer", who);
  IL_CHECK(d >= 1 && d <= IL_GP_MAX_D, "%s: d=%d must be in [1, IL_GP_MAX_D=%d]", who, d, IL_GP_MAX_D);
  IL_CHECK(isfinite(outputscale) && outputscale > 0.0, "%s: outputscale must be finite and > 0 (got %g)", who, outputscale);
  IL_CHECK(isfinite(noise) && noise >= 0.0, "%s: noise must be finite and >= 0 (got %g)", who, noise);
  for (int k = 0; k < IL_GP_MAX_D; ++k) hp->inv_ls[k] = 0.0;
  for (int k = 0; k < d; ++k) {
    IL_CHECK(isfinite(lengthscales[k]) && lengthscales[k] > 0.0, "%s: lengthscale %d must be finite and > 0 (got %g)", who, k, lengthscales[k]);
    hp->inv_ls[k] = 1.0 / lengthscales[k];
  }
  hp->s2 = outputscale;
  hp->noise = noise;
  return 0;
}

}  // namespace

extern "C" int il_gp_posterior(il_handle* h, const double* X, const double* alpha, const double* L, int n, int d, const double* Ct, int64_t M,
                               const double* lengthscales, double outputscale, double noise, double* mu, double* var, double* V, void* stream) {
  IL_CHECK(h && X && alpha && L && Ct && mu && var && V, "il_gp_posterior: null pointer");
  IL_CHECK(n >= 1 && n <= IL_GP_MAX_N, "il_gp_posterior: n=%d must be in [1, IL_GP_MAX_N=%d]", n, IL_GP_MAX_N);
  IL_CHECK(M >= 1 && M <= IL_GP_MAX_M, "il_gp_posterior: M=%lld must be in [1, IL_GP_MAX_M=%d]", (long long)M, IL_GP_MAX_M);
  GpHyper hp;
  IL_TRY(make_hyper(lengthscales, d, outputscale, noise, &hp, "il_gp_posterior"));
  IL_LAUNCH(h, gp_posterior_kernel, (unsigned)((M + POST_THREADS - 1) / POST_THREADS), POST_THREADS, 0, stream, X, alpha, L, n, d, Ct, M, hp, mu, var, V);
  return 0;
}

extern "C" int64_t il_gp_select_workspace_bytes(int n, int d, int64_t M, int q) {
  if (n < 1 || n > IL_GP_MAX_N || d < 1 || d > IL_GP_MAX_D || M < 1 || M > IL_GP_MAX_M || q < 1 || q > IL_GP_MAX_Q || q > M) return -1;
  return sel_layout(n, d, M, q).total;
}

extern "C" int il_gp_select(il_handle* h, int n, int d, const double* Ct, int64_t M, const double* lengthscales, double outputscale, double noise, const double* mu,
                            double* var, double* V, const int32_t* group, int max_groups, double f_star, int q, int32_t* picks, double* ei, void* workspace,
                            int64_t workspace_bytes, void* stream) {
  IL_CHECK(h && Ct && mu && var && V && group && picks && ei && workspace, "il_gp_select: null pointer");
  IL_CHECK(n >= 1 && n <= IL_GP_MAX_N, "il_gp_select: n=%d must be in [1, IL_GP_MAX_N=%d]", n, IL_GP_MAX_N);
  IL_CHECK(M >= 1 && M <= IL_GP_MAX_M, "il_gp_select: M=%lld must be in [1, IL_GP_MAX_M=%d]", (long long)M, IL_GP_MAX_M);
  IL_CHECK(q >= 1 && q <= IL_GP_MAX_Q && q <= M, "il_gp_select: q=%d must be in [1, min(M, IL_GP_MAX_Q=%d)]", q, IL_GP_MAX_Q);
  IL_CHECK(max_groups >= 0, "il_gp_select: max_groups=%d must be >= 0 (0: unlimited)", max_groups);
  IL_CHECK(isfinite(f_star), "il_gp_select: f_star must be finite (got %g)", f_star);
  GpHyper hp;
  IL_TRY(make_hyper(lengthscales, d, outputscale, noise, &hp, "il_gp_select"));
  IL_CHECK(hp.noise > 0.0, "il_gp_select: the kriging-believer update needs noise > 0");
  const SelLayout s = sel_layout(n, d, M, q);
  IL_CHECK(workspace_bytes >= s.total, "il_gp_select: workspace of %lld bytes, need %lld", (long long)workspace_bytes, (long long)s.total);
  char* ws = (char*)workspace;
  int32_t* picked = (int32_t*)(ws + s.picked);
  int32_t* admitted = (int32_t*)(ws + s.admitted);
  SelState* st = (SelState*)(ws + s.state);
  double* vw = (double*)(ws + s.vw);
  double* xw = (double*)(ws + s.xw);
  double* part_v = (double*)(ws + s.part_v);
  int64_t* part_i = (int64_t*)(ws + s.part_i);
  const unsigned nb = (unsigned)((M + SEL_THREADS - 1) / SEL_THREADS);
  IL_LAUNCH(h, gp_select_init_kernel, nb, SEL_THREADS, 0, stream, M, f_star, picked, st);
  IL_LAUNCH(h, gp_select_pass_kernel, nb, SEL_THREADS, 0, stream, M, d, n, hp, Ct, mu, var, V, group, max_groups, picked, admitted, st, vw, xw, 1, part_v, part_i);
  for (int j = 0; j < q; ++j) {
    IL_LAUNCH(h, gp_select_pick_kernel, 1, RED_THREADS, 0, stream, (int)nb, M, d, n + j, part_v, part_i, Ct, mu, var, V, group, max_groups, picked, admitted, st, vw, xw, j,
              picks, ei);
    IL_LAUNCH(h, gp_select_pass_kernel, nb, SEL_THREADS, 0, stream, M, d, n + j, hp, Ct, mu, var, V, group, max_groups, picked, admitted, st, vw, xw, 0, part_v, part_i);
  }
  return 0;
}
