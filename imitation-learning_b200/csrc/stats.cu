// Post-hoc statistics of a seed sweep (scripts/print_plot_seed_sweep_results.py of the reference, printing half): scipy's 25 %-trimmed mean
// (the interquartile mean, IQM), rliable's stratified bootstrap of the IQM over runs x envs, and numpy's linear-interpolation percentiles of
// the bootstrap distribution. All arithmetic is fp64; every sum runs in an order fixed by the launch shape, so results repeat bit for bit.
#include "common.cuh"

namespace {

constexpr int IQM_THREADS = 256;
constexpr int PREP_THREADS = 256;
constexpr int BOOT_THREADS = 256;
constexpr int SMALL_N = 256;  // N up to this: one warp per (rep, t), 8 per block; above: one 256-thread block per (rep, t)
constexpr int SELECT_THREADS = 256;

// Order-preserving map of a double to an unsigned key: a total order equal to numpy's sort order, every NaN above +inf (keys of NaNs are
// equal, so their ties break by index). Ranking on keys, not on `<`, gives every element a distinct rank whatever the input.
__device__ __forceinline__ uint64_t order_key(double v) {
  if (v != v) return ~0ull;
  const uint64_t u = (uint64_t)__double_as_longlong(v);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double from_order_key(uint64_t k) {
  return __longlong_as_double((long long)((k >> 63) ? (k ^ 0x8000000000000000ull) : ~k));
}

// scipy.stats.trim_mean(x, 0.25): order statistics [lc, uc) with lc = floor(n / 4) (int(0.25 * n) is exact in fp64), uc = n - lc
__host__ __device__ inline int iqm_lc(int n) { return n / 4; }

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;  // lane 0 holds the sum
}

// Sum over a block (any blockDim <= 1024) in a fixed tree order; the result is valid in thread 0. red: >= 32 doubles of shared memory.
__device__ double block_sum_d(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum_d(v);
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < nw; ++w) r += red[w];
  return r;
}

// il_iqm: one block per group; the group's order keys are staged in shared memory and each element's stable rank (keys below it, plus
// equal keys at lower indices) decides whether it is inside the window. The kept values are summed by element index (fixed order), not by
// rank: the same multiset, in an order fixed by the input.
__global__ void __launch_bounds__(IQM_THREADS) iqm_kernel(const double* __restrict__ x, int n, double* __restrict__ out) {
  extern __shared__ uint64_t skey[];
  __shared__ double red[32];
  const double* g = x + (int64_t)blockIdx.x * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) skey[i] = order_key(g[i]);
  __syncthreads();
  const int lc = iqm_lc(n), uc = n - lc;
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const uint64_t v = skey[i];
    int r = 0;
    for (int j = 0; j < n; ++j) {
      const uint64_t u = skey[j];
      r += (u < v) || (u == v && j < i);
    }
    if (r >= lc && r < uc) acc += g[i];
  }
  const double s = block_sum_d(acc, red);
  if (threadIdx.x == 0) out[blockIdx.x] = s / (double)(uc - lc);
}

// Bootstrap set-up, once per call: per evaluation point t, the stable sort of its N = envs x runs values (flat index e * runs + r), as
// sorted[t][k] (the k-th smallest value) and perm[t][k] (its flat index). Grid (T, ceil(N / 256)); each thread ranks one element's order
// key against the group's, read through shared-memory tiles.
__global__ void __launch_bounds__(PREP_THREADS) bootstrap_prep_kernel(const double* __restrict__ scores, int N, double* __restrict__ sorted, int32_t* __restrict__ perm) {
  __shared__ uint64_t tile[PREP_THREADS];
  const double* x = scores + (int64_t)blockIdx.x * N;
  const int i = blockIdx.y * PREP_THREADS + threadIdx.x;
  const uint64_t v = i < N ? order_key(x[i]) : 0;
  int r = 0;
  for (int j0 = 0; j0 < N; j0 += PREP_THREADS) {
    __syncthreads();
    if (j0 + threadIdx.x < N) tile[threadIdx.x] = order_key(x[j0 + threadIdx.x]);
    __syncthreads();
    const int m = min(PREP_THREADS, N - j0);
    for (int j = 0; j < m; ++j) {
      const uint64_t u = tile[j];
      r += (u < v) || (u == v && j0 + j < i);
    }
  }
  if (i < N) {  // ranks on the total key order are a permutation of [0, N): every slot is written once
    sorted[(int64_t)blockIdx.x * N + r] = x[i];
    perm[(int64_t)blockIdx.x * N + r] = i;
  }
}

// Exclusive prefix sum over a team of TEAM threads (a warp, or the whole block when TEAM == blockDim.x); also returns the team total.
// scratch: TEAM / 32 ints of shared memory owned by the team (unused for a warp).
template <int TEAM>
__device__ __forceinline__ int team_exclusive_scan(int v, int* scratch, int& total) {
  const int lane = threadIdx.x & 31;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (TEAM == 32) {
    total = __shfl_sync(0xffffffffu, inc, 31);
    return inc - v;
  }
  const int warp = (threadIdx.x % TEAM) >> 5;
  if (lane == 31) scratch[warp] = inc;
  __syncthreads();
  int before = 0;
  total = 0;
#pragma unroll
  for (int w = 0; w < TEAM / 32; ++w) {
    const int s = scratch[w];
    if (w < warp) before += s;
    total += s;
  }
  __syncthreads();
  return before + inc - v;
}

// Team sum in a fixed tree order, valid in the team's first thread. scratch: TEAM / 32 doubles (unused for a warp).
template <int TEAM>
__device__ __forceinline__ double team_sum(double v, double* scratch) {
  v = warp_sum_d(v);
  if (TEAM == 32) return v;
  const int lane = threadIdx.x & 31, warp = (threadIdx.x % TEAM) >> 5;
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x % TEAM == 0)
#pragma unroll
    for (int w = 0; w < TEAM / 32; ++w) r += scratch[w];
  return r;
}

__device__ __forceinline__ void team_sync(int team) {
  if (team == 32) __syncwarp();
  else __syncthreads();
}

// One (rep, t) per team of TEAM threads. The resample only changes how many times each of the N values is taken, so the team builds that
// multiplicity as an integer histogram over flat indices in shared memory, then walks the values in sorted order once: with c the number of
// resampled values below slot k and m its multiplicity, the slot contributes (clamp(c + m) - clamp(c)) x sorted[k], clamp to [lc, uc).
// Each thread owns a contiguous run of slots, so the sum order is fixed. A histogram whose total is not N (an out-of-range injected index)
// yields NaN.
template <int TEAM>
__global__ void __launch_bounds__(BOOT_THREADS) bootstrap_iqm_kernel(const double* __restrict__ sorted, const int32_t* __restrict__ perm, int T, int envs, int runs,
                                                                     int64_t pairs, uint64_t seed, const int32_t* __restrict__ indices, double* __restrict__ out) {
  constexpr int TEAMS = BOOT_THREADS / TEAM;
  extern __shared__ int hist_all[];
  __shared__ int iscratch[BOOT_THREADS / 32];
  __shared__ double dscratch[BOOT_THREADS / 32];
  const int N = envs * runs;
  const int team = threadIdx.x / TEAM, tl = threadIdx.x % TEAM;
  const int64_t p = (int64_t)blockIdx.x * TEAMS + team;  // p = rep * T + t
  if (TEAM == 32 && p >= pairs) return;                  // whole warps only; the block-team launch has exactly `pairs` blocks
  int* hist = hist_all + team * N;
  const int rep = (int)(p / T), t = (int)(p % T);
  for (int s = tl; s < N; s += TEAM) hist[s] = 0;
  team_sync(TEAM);
  if (indices) {
    const int32_t* idx = indices + p * N;
    for (int d = tl; d < N; d += TEAM) {
      const int r = idx[d];
      if ((unsigned)r < (unsigned)runs) atomicAdd(&hist[(d / runs) * runs + r], 1);
    }
  } else {
    // draw k of (rep, t, env e) is lane k % 4 of Philox4x32-10(counter (k / 4, e, t, rep), key seed), mapped to a run by (u * runs) >> 32
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    const int Q = (runs + 3) / 4;
    for (int q = tl; q < envs * Q; q += TEAM) {
      const int e = q / Q, k0 = (q % Q) * 4;
      const uint4 u = philox4x32_10(make_uint4((uint32_t)(k0 / 4), (uint32_t)e, (uint32_t)t, (uint32_t)rep), key);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (k0 + c < runs) atomicAdd(&hist[e * runs + (int)(((uint64_t)w[c] * (uint32_t)runs) >> 32)], 1);
    }
  }
  team_sync(TEAM);
  const double* sv = sorted + (int64_t)t * N;
  const int32_t* pv = perm + (int64_t)t * N;
  const int chunk = (N + TEAM - 1) / TEAM, s0 = min(N, tl * chunk), s1 = min(N, s0 + chunk);
  int local = 0;
  for (int s = s0; s < s1; ++s) local += hist[pv[s]];
  int total;
  int c = team_exclusive_scan<TEAM>(local, iscratch + team * (TEAM / 32), total);
  const int lc = iqm_lc(N), uc = N - lc;
  double acc = 0.0;
  for (int s = s0; s < s1; ++s) {
    const int m = hist[pv[s]];
    const int w = min(max(c + m, lc), uc) - min(max(c, lc), uc);
    if (w) acc += (double)w * sv[s];
    c += m;
  }
  const double sum = team_sum<TEAM>(acc, dscratch + team * (TEAM / 32));
  if (tl == 0) out[p] = total == N ? sum / (double)(uc - lc) : __longlong_as_double(0x7ff8000000000000ll);
}

// k-th smallest (0-based) of x[i * stride], i < n, by an 8-bit MSB-first radix select; called by the whole block.
__device__ double block_select(const double* x, int64_t n, int stride, int64_t k, unsigned* hist, uint64_t* sh) {
  uint64_t prefix = 0, mask = 0;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0;
    __syncthreads();
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const uint64_t key = order_key(x[i * stride]);
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int64_t below = 0;
      int b = 0;
      for (; b < 255 && k >= below + hist[b]; ++b) below += hist[b];
      sh[0] = prefix | ((uint64_t)b << shift);
      sh[1] = (uint64_t)(k - below);
    }
    __syncthreads();
    prefix = sh[0];
    k = (int64_t)sh[1];
    mask |= 0xffull << shift;
    __syncthreads();
  }
  return from_order_key(prefix);
}

// numpy.percentile(x, pct) with the default 'linear' method, step for step: virtual index (n - 1) (pct / 100), neighbours clipped to
// [0, n - 1], and numpy's two-sided lerp (b - (b - a)(1 - g) where g >= 0.5).
__device__ double block_percentile(const double* x, int64_t n, int stride, double pct, unsigned* hist, uint64_t* sh) {
  const double virt = (double)(n - 1) * (pct / 100.0);
  const double prev = floor(virt);
  const double g = virt - prev;
  int64_t lo, hi;
  if (virt >= (double)(n - 1)) lo = hi = n - 1;
  else if (virt < 0.0) lo = hi = 0;
  else lo = (int64_t)prev, hi = lo + 1;
  const double a = block_select(x, n, stride, lo, hist, sh);
  const double b = hi == lo ? a : block_select(x, n, stride, hi, hist, sh);
  const double d = b - a;
  return g >= 0.5 ? __dsub_rn(b, __dmul_rn(d, 1.0 - g)) : __dadd_rn(a, __dmul_rn(d, g));  // unfused, as numpy rounds them
}

// One block per evaluation point t: out[0][t], out[1][t] = the q_lo and q_hi percentiles of the column dist[:, t] of dist [reps, T].
__global__ void __launch_bounds__(SELECT_THREADS) percentile_interval_kernel(const double* __restrict__ dist, int reps, int T, double q_lo, double q_hi, double* __restrict__ out) {
  __shared__ unsigned hist[256];
  __shared__ uint64_t sh[2];
  const int t = blockIdx.x;
  const double lo = block_percentile(dist + t, reps, T, q_lo, hist, sh);
  const double hi = block_percentile(dist + t, reps, T, q_hi, hist, sh);
  if (threadIdx.x == 0) {
    out[t] = lo;
    out[T + t] = hi;
  }
}

}  // namespace

extern "C" int il_iqm(il_handle* h, const double* x, int64_t G, int n, double* out, void* stream) {
  IL_CHECK(h && x && out, "il_iqm: null pointer");
  IL_CHECK(G > 0 && G <= 0x7fffffff && n > 0, "il_iqm: need G > 0 (below 2^31) and n > 0 (got G=%lld, n=%d)", (long long)G, n);
  IL_CHECK(n <= IL_IQM_MAX_N, "il_iqm: n=%d exceeds IL_IQM_MAX_N=%d", n, IL_IQM_MAX_N);
  const size_t smem = (size_t)n * sizeof(uint64_t);
  if (smem > 48 * 1024) IL_CUDA(cudaFuncSetAttribute(iqm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  IL_LAUNCH(h, iqm_kernel, (unsigned)G, IQM_THREADS, smem, (cudaStream_t)stream, x, n, out);
  return 0;
}

extern "C" int64_t il_bootstrap_iqm_workspace_bytes(int T, int envs, int runs) {
  if (T <= 0 || envs <= 0 || runs <= 0 || (int64_t)envs * runs > IL_BOOTSTRAP_MAX_N) return -1;
  const int64_t TN = (int64_t)T * envs * runs;
  return il_align_up(TN * (int64_t)sizeof(double), 256) + il_align_up(TN * (int64_t)sizeof(int32_t), 256);
}

extern "C" int il_bootstrap_iqm(il_handle* h, const double* scores, int T, int envs, int runs, int reps, uint64_t seed, const int32_t* indices, double* out,
                                void* workspace, int64_t workspace_bytes, void* stream) {
  IL_CHECK(h && scores && out && workspace, "il_bootstrap_iqm: null pointer");
  IL_CHECK(T > 0 && envs > 0 && runs > 0 && reps > 0, "il_bootstrap_iqm: sizes must be positive (T=%d, envs=%d, runs=%d, reps=%d)", T, envs, runs, reps);
  const int64_t N64 = (int64_t)envs * runs;
  IL_CHECK(N64 <= IL_BOOTSTRAP_MAX_N, "il_bootstrap_iqm: envs x runs = %lld exceeds IL_BOOTSTRAP_MAX_N=%d", (long long)N64, IL_BOOTSTRAP_MAX_N);
  const int64_t pairs = (int64_t)reps * T;
  IL_CHECK(pairs <= 0x7fffffff, "il_bootstrap_iqm: reps x T = %lld must stay below 2^31", (long long)pairs);
  const int64_t need = il_bootstrap_iqm_workspace_bytes(T, envs, runs);
  IL_CHECK(workspace_bytes >= need, "il_bootstrap_iqm: workspace of %lld bytes, need %lld", (long long)workspace_bytes, (long long)need);
  const int N = (int)N64;
  const int64_t TN = (int64_t)T * N;
  double* sorted = (double*)workspace;
  int32_t* perm = (int32_t*)((char*)workspace + il_align_up(TN * (int64_t)sizeof(double), 256));
  cudaStream_t st = (cudaStream_t)stream;
  IL_LAUNCH(h, bootstrap_prep_kernel, dim3((unsigned)T, (unsigned)((N + PREP_THREADS - 1) / PREP_THREADS)), PREP_THREADS, 0, st, scores, N, sorted, perm);
  if (N <= SMALL_N) {
    constexpr int TEAMS = BOOT_THREADS / 32;
    IL_LAUNCH(h, bootstrap_iqm_kernel<32>, (unsigned)((pairs + TEAMS - 1) / TEAMS), BOOT_THREADS, (size_t)TEAMS * N * sizeof(int), st, sorted, perm, T, envs, runs, pairs, seed,
              indices, out);
  } else {
    IL_LAUNCH(h, bootstrap_iqm_kernel<BOOT_THREADS>, (unsigned)pairs, BOOT_THREADS, (size_t)N * sizeof(int), st, sorted, perm, T, envs, runs, pairs, seed, indices, out);
  }
  return 0;
}

extern "C" int il_percentile_interval(il_handle* h, const double* dist, int reps, int T, double q_lo, double q_hi, double* out2, void* stream) {
  IL_CHECK(h && dist && out2, "il_percentile_interval: null pointer");
  IL_CHECK(reps > 0 && T > 0, "il_percentile_interval: sizes must be positive (reps=%d, T=%d)", reps, T);
  IL_CHECK(q_lo >= 0.0 && q_lo <= 100.0 && q_hi >= 0.0 && q_hi <= 100.0, "il_percentile_interval: percentiles must lie in [0, 100] (got %g, %g)", q_lo, q_hi);
  IL_LAUNCH(h, percentile_interval_kernel, (unsigned)T, SELECT_THREADS, 0, (cudaStream_t)stream, dist, reps, T, q_lo, q_hi, out2);
  return 0;
}
