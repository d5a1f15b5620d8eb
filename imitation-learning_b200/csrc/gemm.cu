// Grouped fp32 GEMM with fused MLP epilogues (bias, activation, activation-derivative mask, bias-gradient
// column sums). One launch covers all replicas (groups): the reference's per-network nn.Linear forward /
// autograd backward (models.py:48-69 as used by training.py:14-54) batched over the replica axis.
//
// This is the exact-fp32 (FFMA) engine. The dense H x H layers can instead be routed to the wgmma engine
// (tc_gemm.cu) by il_set_gemm_mode; everything thin (K = state size, N = 1 or 2A) stays here.
#include "common.cuh"

namespace {

template <int V>
__device__ __forceinline__ void lds_vec(float* dst, const float* src) {
  if constexpr (V == 4) {
    const float4 t = *reinterpret_cast<const float4*>(src);
    dst[0] = t.x; dst[1] = t.y; dst[2] = t.z; dst[3] = t.w;
  } else if constexpr (V == 2) {
    const float2 t = *reinterpret_cast<const float2*>(src);
    dst[0] = t.x; dst[1] = t.y;
  } else {
    dst[0] = src[0];
  }
}

template <int BM, int BN, int BK, int TM, int TN, bool A_KMAJOR, bool B_KMAJOR>
__global__ void __launch_bounds__(256, 2) gemm_grouped_kernel(const GemmArgs p) {
  constexpr int THREADS = 256;
  static_assert((BM / TM) * (BN / TN) == THREADS, "tile/thread mismatch");
  constexpr int VM = TM >= 4 ? 4 : TM, VN = TN >= 4 ? 4 : TN;
  constexpr int RC = TM / VM, CC = TN / VN;
  constexpr int LDAS = BM + 4, LDBS = BN + 4;
  constexpr int A_F4 = BM * BK / 4, B_F4 = BN * BK / 4;
  constexpr int LA = (A_F4 + THREADS - 1) / THREADS, LB = (B_F4 + THREADS - 1) / THREADS;

  __shared__ __align__(16) float As[2][BK][LDAS];
  __shared__ __align__(16) float Bs[2][BK][LDBS];

  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int g = blockIdx.z;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int M = p.M, N = p.N, K = p.K;

  const float* __restrict__ A = p.A + (int64_t)(g / p.a_gdiv) * p.a_gs;
  const float* __restrict__ B = p.B + (int64_t)(g / p.b_gdiv) * p.b_gs;
  const bool vecA = ((reinterpret_cast<uintptr_t>(p.A) & 15) == 0) && (p.a_gs % 4 == 0) && (p.lda % 4 == 0);
  const bool vecB = ((reinterpret_cast<uintptr_t>(p.B) & 15) == 0) && (p.b_gs % 4 == 0) && (p.ldb % 4 == 0);

  float4 ra[LA], rb[LB];
  float4 csum = make_float4(0.f, 0.f, 0.f, 0.f);
  const bool do_colsum = (!A_KMAJOR) && (p.colsum != nullptr) && (blockIdx.x == 0);

  auto load_a = [&](int k0) {
#pragma unroll
    for (int j = 0; j < LA; ++j) {
      const int i = tid + j * THREADS;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i < A_F4) {
        if constexpr (A_KMAJOR) {
          const int row = m0 + i / (BK / 4), kq = k0 + (i % (BK / 4)) * 4;
          if (row < M) {
            const float* src = A + (int64_t)row * p.lda + kq;
            if (vecA && kq + 3 < K) {
              v = __ldg(reinterpret_cast<const float4*>(src));
            } else {
              if (kq + 0 < K) v.x = __ldg(src + 0);
              if (kq + 1 < K) v.y = __ldg(src + 1);
              if (kq + 2 < K) v.z = __ldg(src + 2);
              if (kq + 3 < K) v.w = __ldg(src + 3);
            }
          }
        } else {
          const int kr = k0 + i / (BM / 4), mq = m0 + (i % (BM / 4)) * 4;
          if (kr < K) {
            const float* src = A + (int64_t)kr * p.lda + mq;
            if (vecA && mq + 3 < M) {
              v = __ldg(reinterpret_cast<const float4*>(src));
            } else {
              if (mq + 0 < M) v.x = __ldg(src + 0);
              if (mq + 1 < M) v.y = __ldg(src + 1);
              if (mq + 2 < M) v.z = __ldg(src + 2);
              if (mq + 3 < M) v.w = __ldg(src + 3);
            }
          }
        }
      }
      ra[j] = v;
    }
  };
  auto load_b = [&](int k0) {
#pragma unroll
    for (int j = 0; j < LB; ++j) {
      const int i = tid + j * THREADS;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i < B_F4) {
        if constexpr (B_KMAJOR) {
          const int row = n0 + i / (BK / 4), kq = k0 + (i % (BK / 4)) * 4;
          if (row < N) {
            const float* src = B + (int64_t)row * p.ldb + kq;
            if (vecB && kq + 3 < K) {
              v = __ldg(reinterpret_cast<const float4*>(src));
            } else {
              if (kq + 0 < K) v.x = __ldg(src + 0);
              if (kq + 1 < K) v.y = __ldg(src + 1);
              if (kq + 2 < K) v.z = __ldg(src + 2);
              if (kq + 3 < K) v.w = __ldg(src + 3);
            }
          }
        } else {
          const int kr = k0 + i / (BN / 4), nq = n0 + (i % (BN / 4)) * 4;
          if (kr < K) {
            const float* src = B + (int64_t)kr * p.ldb + nq;
            if (vecB && nq + 3 < N) {
              v = __ldg(reinterpret_cast<const float4*>(src));
            } else {
              if (nq + 0 < N) v.x = __ldg(src + 0);
              if (nq + 1 < N) v.y = __ldg(src + 1);
              if (nq + 2 < N) v.z = __ldg(src + 2);
              if (nq + 3 < N) v.w = __ldg(src + 3);
            }
          }
        }
      }
      rb[j] = v;
    }
  };
  auto store_a = [&](int buf) {
#pragma unroll
    for (int j = 0; j < LA; ++j) {
      const int i = tid + j * THREADS;
      if (i < A_F4) {
        if constexpr (A_KMAJOR) {
          const int row = i / (BK / 4), kq = (i % (BK / 4)) * 4;
          As[buf][kq + 0][row] = ra[j].x;
          As[buf][kq + 1][row] = ra[j].y;
          As[buf][kq + 2][row] = ra[j].z;
          As[buf][kq + 3][row] = ra[j].w;
        } else {
          const int kr = i / (BM / 4), mq = (i % (BM / 4)) * 4;
          *reinterpret_cast<float4*>(&As[buf][kr][mq]) = ra[j];
          if (do_colsum) { csum.x += ra[j].x; csum.y += ra[j].y; csum.z += ra[j].z; csum.w += ra[j].w; }
        }
      }
    }
  };
  auto store_b = [&](int buf) {
#pragma unroll
    for (int j = 0; j < LB; ++j) {
      const int i = tid + j * THREADS;
      if (i < B_F4) {
        if constexpr (B_KMAJOR) {
          const int row = i / (BK / 4), kq = (i % (BK / 4)) * 4;
          Bs[buf][kq + 0][row] = rb[j].x;
          Bs[buf][kq + 1][row] = rb[j].y;
          Bs[buf][kq + 2][row] = rb[j].z;
          Bs[buf][kq + 3][row] = rb[j].w;
        } else {
          const int kr = i / (BN / 4), nq = (i % (BN / 4)) * 4;
          *reinterpret_cast<float4*>(&Bs[buf][kr][nq]) = rb[j];
        }
      }
    }
  };

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nk = (K + BK - 1) / BK;
  load_a(0);
  load_b(0);
  store_a(0);
  store_b(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) {
      load_a((kt + 1) * BK);
      load_b((kt + 1) * BK);
    }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int rc = 0; rc < RC; ++rc) lds_vec<VM>(&a[rc * VM], &As[buf][k][rc * (BM / RC) + ty * VM]);
#pragma unroll
      for (int cc = 0; cc < CC; ++cc) lds_vec<VN>(&b[cc * VN], &Bs[buf][k][cc * (BN / CC) + tx * VN]);
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_a(buf ^ 1);
      store_b(buf ^ 1);
    }
    __syncthreads();
  }

  // ---- epilogue ----
  float* __restrict__ C = p.C + (int64_t)g * p.c_gs;
  const float* __restrict__ bias = p.bias ? p.bias + (int64_t)g * p.bias_gs : nullptr;
  const float* __restrict__ mask = p.mask ? p.mask + (int64_t)g * p.mask_gs : nullptr;
#pragma unroll
  for (int rc = 0; rc < RC; ++rc) {
#pragma unroll
    for (int i = 0; i < VM; ++i) {
      const int m = m0 + rc * (BM / RC) + ty * VM + i;
      if (m >= M) continue;
#pragma unroll
      for (int cc = 0; cc < CC; ++cc) {
#pragma unroll
        for (int j = 0; j < VN; ++j) {
          const int n = n0 + cc * (BN / CC) + tx * VN + j;
          if (n >= N) continue;
          float v = acc[rc * VM + i][cc * VN + j];
          if (bias) v += __ldg(bias + n);
          if (p.accumulate) v += C[(int64_t)m * p.ldc + n];
          if (p.act >= 0) v = act_apply(v, p.act);
          if (mask) v *= act_grad_from_output(__ldg(mask + (int64_t)m * p.ldmask + n), p.mask_act);
          C[(int64_t)m * p.ldc + n] = v;
        }
      }
    }
  }

  if constexpr (!A_KMAJOR) {
    if (do_colsum) {  // bias gradient: colsum[m] = sum_k A[k, m], deterministic order
      constexpr int ACTIVE = A_F4 < THREADS ? A_F4 : THREADS;  // threads that loaded A
      static_assert(ACTIVE * 4 <= 2 * BK * LDAS, "colsum partials do not fit in As");
      float4* red = reinterpret_cast<float4*>(&As[0][0][0]);
      if (tid < ACTIVE) red[tid] = csum;  // only these slots are read back; 256 float4 would overrun As for BM = 16
      __syncthreads();
      if (tid < BM && m0 + tid < M) {
        constexpr int CH = BM / 4;  // float4 chunks per k row
        const int chunk = tid / 4, comp = tid % 4;
        float s = 0.f;
        for (int t = chunk; t < ACTIVE; t += CH) s += reinterpret_cast<const float*>(&red[t])[comp];
        p.colsum[(int64_t)g * p.colsum_gs + m0 + tid] = s;
      }
    }
  }
}

// Thin-contraction kernel (K <= 32, wide output): the first layer of every MLP (K = state size) and the backward of
// the last layer (K = head width). These products are pure output bandwidth, so the tile loop of the general kernel is
// replaced by: B (K x 256) and 32 rows of A in shared memory, 8 x 4 outputs per thread, 128-bit coalesced stores.
constexpr int TK_MAXK = 32, TK_ROWS = 32, TK_ITERS = 4, TK_COLS = 256, TK_LDA = TK_MAXK + 4;  // a CTA covers 4 x 32 rows
// (8 x 32 rows per CTA with a coalesced, bank-spread staging of the [N, K] weights was not faster on the whole step.)
// HOIST_MASK: the activation-derivative mask rows of an iteration are loaded before the FMA loop (8 x 128-bit loads in
// flight per thread, 2 CTAs/SM) instead of one by one inside the store loop (the masked variant is latency-bound).
template <bool B_KMAJOR, bool HOIST_MASK>
__global__ void __launch_bounds__(256, HOIST_MASK ? 2 : 3) gemm_thin_k_kernel(const GemmArgs p) {
  __shared__ __align__(16) float Bs[TK_MAXK][TK_COLS];
  __shared__ __align__(16) float As[TK_ROWS][TK_LDA];  // K zero-padded to a multiple of 4 so rows are read as float4
  const int tid = threadIdx.x, g = blockIdx.z, n0 = blockIdx.x * TK_COLS;
  const int M = p.M, N = p.N, K = p.K, K4 = (K + 3) & ~3;
  const float* __restrict__ A = p.A + (int64_t)(g / p.a_gdiv) * p.a_gs;
  const float* __restrict__ B = p.B + (int64_t)(g / p.b_gdiv) * p.b_gs;
  const int ncols = min(TK_COLS, N - n0);
  // B (K x ncols) staged once per CTA; consecutive threads -> consecutive n (conflict-free shared stores; the strided
  // global reads of the [N, K] weight layout stay in L1/L2: the whole matrix is K * N * 4 <= 32 KB)
  for (int idx = tid; idx < K4 * TK_COLS; idx += 256) {
    const int k = idx / TK_COLS, n = idx % TK_COLS;
    float v = 0.f;
    if (k < K && n < ncols) v = B_KMAJOR ? __ldg(B + (int64_t)(n0 + n) * p.ldb + k) : __ldg(B + (int64_t)k * p.ldb + n0 + n);
    Bs[k][n] = v;
  }
  const int n = (tid & 63) * 4, tr = tid >> 6;
  float* __restrict__ C = p.C + (int64_t)g * p.c_gs;
  const float* __restrict__ mask = p.mask ? p.mask + (int64_t)g * p.mask_gs : nullptr;
  float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
  if (p.bias && n < ncols) bv = __ldg(reinterpret_cast<const float4*>(p.bias + (int64_t)g * p.bias_gs + n0 + n));
  // A rows of the next 32-row block are fetched into registers while the current block is computed
  constexpr int A_PER = TK_ROWS * TK_MAXK / 256;  // 4 elements per thread cover the zero-padded [32][K4 <= 32] tile
  float a_next[A_PER];
  auto fetch_a = [&](int m0) {
#pragma unroll
    for (int q = 0; q < A_PER; ++q) {
      const int idx = tid + q * 256, r = idx / K4, k = idx % K4;
      a_next[q] = (idx < TK_ROWS * K4 && m0 + r < M && k < K) ? __ldg(A + (int64_t)(m0 + r) * p.lda + k) : 0.f;
    }
  };
  fetch_a(blockIdx.y * TK_ITERS * TK_ROWS);
  for (int it = 0; it < TK_ITERS; ++it) {
    const int m0 = (blockIdx.y * TK_ITERS + it) * TK_ROWS;
    if (m0 >= M) break;
    __syncthreads();  // previous iteration's readers of As are done (and Bs is complete on the first pass)
#pragma unroll
    for (int q = 0; q < A_PER; ++q) {
      const int idx = tid + q * 256;
      if (idx < TK_ROWS * K4) As[idx / K4][idx % K4] = a_next[q];
    }
    __syncthreads();
    if (it + 1 < TK_ITERS && m0 + TK_ROWS < M) fetch_a(m0 + TK_ROWS);
    if (n >= ncols) continue;
    float4 mvh[HOIST_MASK ? 8 : 1];
    if (HOIST_MASK) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int m = m0 + tr + 4 * i;
        mvh[i] = m < M ? __ldg(reinterpret_cast<const float4*>(mask + (int64_t)m * p.ldmask + n0 + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    for (int k = 0; k < K4; k += 4) {
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[k][n]), b1 = *reinterpret_cast<const float4*>(&Bs[k + 1][n]);
      const float4 b2 = *reinterpret_cast<const float4*>(&Bs[k + 2][n]), b3 = *reinterpret_cast<const float4*>(&Bs[k + 3][n]);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 a = *reinterpret_cast<const float4*>(&As[tr + 4 * i][k]);  // warp-uniform address: one broadcast load for 4 k
        acc[i][0] = fmaf(a.x, b0.x, acc[i][0]); acc[i][1] = fmaf(a.x, b0.y, acc[i][1]); acc[i][2] = fmaf(a.x, b0.z, acc[i][2]); acc[i][3] = fmaf(a.x, b0.w, acc[i][3]);
        acc[i][0] = fmaf(a.y, b1.x, acc[i][0]); acc[i][1] = fmaf(a.y, b1.y, acc[i][1]); acc[i][2] = fmaf(a.y, b1.z, acc[i][2]); acc[i][3] = fmaf(a.y, b1.w, acc[i][3]);
        acc[i][0] = fmaf(a.z, b2.x, acc[i][0]); acc[i][1] = fmaf(a.z, b2.y, acc[i][1]); acc[i][2] = fmaf(a.z, b2.z, acc[i][2]); acc[i][3] = fmaf(a.z, b2.w, acc[i][3]);
        acc[i][0] = fmaf(a.w, b3.x, acc[i][0]); acc[i][1] = fmaf(a.w, b3.y, acc[i][1]); acc[i][2] = fmaf(a.w, b3.z, acc[i][2]); acc[i][3] = fmaf(a.w, b3.w, acc[i][3]);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int m = m0 + tr + 4 * i;
      if (m >= M) continue;
      float4 v = make_float4(acc[i][0] + bv.x, acc[i][1] + bv.y, acc[i][2] + bv.z, acc[i][3] + bv.w);
      if (p.act >= 0) { v.x = act_apply(v.x, p.act); v.y = act_apply(v.y, p.act); v.z = act_apply(v.z, p.act); v.w = act_apply(v.w, p.act); }
      if (mask) {
        const float4 mv = HOIST_MASK ? mvh[i] : __ldg(reinterpret_cast<const float4*>(mask + (int64_t)m * p.ldmask + n0 + n));
        v.x *= act_grad_from_output(mv.x, p.mask_act); v.y *= act_grad_from_output(mv.y, p.mask_act);
        v.z *= act_grad_from_output(mv.z, p.mask_act); v.w *= act_grad_from_output(mv.w, p.mask_act);
      }
      *reinterpret_cast<float4*>(C + (int64_t)m * p.ldc + n0 + n) = v;
    }
  }
}


// First MLP layer, specialised: C = relu(A W^T + b) with K <= 16 input columns (state or state + action), N a multiple of 256, M a multiple
// of 32. The generic K-thin kernel above is instruction-issue bound on this shape; here the
// contraction runs on two FFMA chains over k-pairs ({a_k, a_k+1} x {w_k, w_k+1} accumulate the even / odd partial sums, added at the end), the
// activation is compile-time and there are no bounds checks in the inner loops: ~3x fewer issued instructions, so the kernel is bound by
// its 128-bit output stores instead.
constexpr int FL_K = 16, FL_ROWS = 32, FL_ITERS = 4, FL_COLS = 256;
// Packed pairs of fp32 travel as one 64-bit register pair (128-bit shared-memory loads deliver two of them); sm_90 has no packed
// fp32 arithmetic, so each half is one IEEE fp32 FMA / multiply.
__device__ __forceinline__ unsigned long long fl_fma2(unsigned long long a, unsigned long long b, unsigned long long c) {
  float ax, ay, bx, by, cx, cy;
  unsigned long long d;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(ax), "=f"(ay) : "l"(a));
  asm("mov.b64 {%0, %1}, %2;" : "=f"(bx), "=f"(by) : "l"(b));
  asm("mov.b64 {%0, %1}, %2;" : "=f"(cx), "=f"(cy) : "l"(c));
  asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "f"(fmaf(ax, bx, cx)), "f"(fmaf(ay, by, cy)));
  return d;
}
__device__ __forceinline__ unsigned long long fl_mul2(unsigned long long a, unsigned long long b) {
  float ax, ay, bx, by;
  unsigned long long d;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(ax), "=f"(ay) : "l"(a));
  asm("mov.b64 {%0, %1}, %2;" : "=f"(bx), "=f"(by) : "l"(b));
  asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "f"(__fmul_rn(ax, bx)), "f"(__fmul_rn(ay, by)));
  return d;
}
__global__ void __launch_bounds__(256, 2) first_layer_relu_kernel(const GemmArgs p) {
  __shared__ __align__(16) float Ws[(FL_K / 2) * FL_COLS * 2];  // [k pair][n][2]
  __shared__ __align__(16) float As[FL_ROWS][FL_K];
  const int tid = threadIdx.x, g = blockIdx.z, n0 = blockIdx.x * FL_COLS, K = p.K;
  const float* __restrict__ A = p.A + (int64_t)(g / p.a_gdiv) * p.a_gs;
  const float* __restrict__ W = p.B + (int64_t)(g / p.b_gdiv) * p.b_gs;
  for (int idx = tid; idx < FL_K * FL_COLS; idx += 256) {
    const int k = idx / FL_COLS, n = idx % FL_COLS;
    Ws[(k >> 1) * (FL_COLS * 2) + n * 2 + (k & 1)] = k < K ? __ldg(W + (int64_t)(n0 + n) * p.ldb + k) : 0.f;
  }
  const int n = (tid & 63) * 4, tr = tid >> 6;
  float* __restrict__ C = p.C + (int64_t)g * p.c_gs + n0 + n;
  const float4 bv = __ldg(reinterpret_cast<const float4*>(p.bias + (int64_t)g * p.bias_gs + n0 + n));
  float a_next[2];
  auto fetch_a = [&](int m0) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int idx = tid + q * 256, r = idx / FL_K, k = idx % FL_K;
      a_next[q] = k < K ? __ldg(A + (int64_t)(m0 + r) * p.lda + k) : 0.f;
    }
  };
  const int mbase = blockIdx.y * FL_ITERS * FL_ROWS;
  fetch_a(mbase);
  for (int it = 0; it < FL_ITERS; ++it) {
    const int m0 = mbase + it * FL_ROWS;
    if (m0 >= p.M) break;
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 2; ++q) { const int idx = tid + q * 256; As[idx / FL_K][idx % FL_K] = a_next[q]; }
    __syncthreads();
    if (it + 1 < FL_ITERS && m0 + FL_ROWS < p.M) fetch_a(m0 + FL_ROWS);
    unsigned long long acc[8][4];  // {even-k partial, odd-k partial} per (row, column)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0ull;
#pragma unroll
    for (int kq = 0; kq < FL_K / 4; ++kq) {  // 4 k's = 2 pairs per step
      unsigned long long w[2][4];
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const ulonglong2 lo = *reinterpret_cast<const ulonglong2*>(&Ws[(kq * 2 + h2) * (FL_COLS * 2) + n * 2]);
        const ulonglong2 hi = *reinterpret_cast<const ulonglong2*>(&Ws[(kq * 2 + h2) * (FL_COLS * 2) + n * 2 + 4]);
        w[h2][0] = lo.x; w[h2][1] = lo.y; w[h2][2] = hi.x; w[h2][3] = hi.y;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const ulonglong2 a = *reinterpret_cast<const ulonglong2*>(&As[tr + 4 * i][kq * 4]);  // {a_k, a_k+1}, {a_k+2, a_k+3}: warp-uniform address
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          acc[i][c] = fl_fma2(a.x, w[0][c], acc[i][c]);
          acc[i][c] = fl_fma2(a.y, w[1][c], acc[i][c]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float e, o;
        asm("mov.b64 {%0, %1}, %2;" : "=f"(e), "=f"(o) : "l"(acc[i][c]));
        v[c] = e + o;
      }
      const float4 out = make_float4(fmaxf(v[0] + bv.x, 0.f), fmaxf(v[1] + bv.y, 0.f), fmaxf(v[2] + bv.z, 0.f), fmaxf(v[3] + bv.w, 0.f));
      *reinterpret_cast<float4*>(C + (int64_t)(m0 + tr + 4 * i) * p.ldc) = out;
    }
  }
}

// Register-resident variant for N == 256 (one CTA = one net's whole [<= 256 rows] x [256 columns] first-layer output): each thread keeps the
// K x 4 weights of its 4 columns packed as k-pairs in registers for all of its rows, the net's input rows sit in shared memory (one stage, one
// barrier), and the row loop has no barriers and only warp-broadcast shared loads: per 2 rows x 4 columns 2*ceil(K/4) LDS.128 + 8*ceil(K/2)
// k-pair FFMA + 2 STG.128. (first_layer_relu_kernel pays two 128-bit shared-memory
// weight loads per 8 k-pair FFMA, per-32-row barriers and a strided weight prologue.) K is a template parameter so the weight registers are
// statically indexed.
template <int K, bool BITS>
__global__ void __launch_bounds__(256, 2) first_layer_reg_kernel(const GemmArgs p) {
  constexpr int KP = (K + 1) / 2, KQ = (K + 3) / 4, LDS_A = KQ * 4;
  // odd K: the zero-padded last k slot carries the bias instead (input 1, weight b): the accumulators start from a product, not from a {bias, 0}
  // register pair that has to be rebuilt (2 MOVs) for each of the 8 accumulators of every iteration
  constexpr bool BIAS_COL = (K % 2) == 1;
  __shared__ __align__(16) float As[256 * LDS_A];
  const int tid = threadIdx.x, g = blockIdx.y, m_base = blockIdx.x * 256;
  const int rows = p.M - m_base < 256 ? p.M - m_base : 256;
  const float* __restrict__ A = p.A + (int64_t)(g / p.a_gdiv) * p.a_gs + (int64_t)m_base * p.lda;
  const float* __restrict__ W = p.B + (int64_t)(g / p.b_gdiv) * p.b_gs;
  const int n = (tid & 63) * 4, tr = tid >> 6;
  if (tid < rows) {  // stage the input rows (zero padded to a multiple of 4 columns)
    const float* ar = A + (int64_t)tid * p.lda;
    float v[LDS_A];
#pragma unroll
    for (int k = 0; k < LDS_A; ++k) v[k] = k < K ? __ldg(ar + k) : ((BIAS_COL && k == K) ? 1.f : 0.f);
#pragma unroll
    for (int q = 0; q < KQ; ++q) *reinterpret_cast<float4*>(&As[tid * LDS_A + 4 * q]) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  }
  const float4 bv = __ldg(reinterpret_cast<const float4*>(p.bias + (int64_t)g * p.bias_gs + n));
  const float bvc[4] = {bv.x, bv.y, bv.z, bv.w};
  unsigned long long w[KP][4];
  {  // rows n .. n + 3 of W [256][K] are 4 K contiguous floats starting on a 16-byte boundary
    float f[4 * K];
    const float4* src = reinterpret_cast<const float4*>(W + (int64_t)n * K);
#pragma unroll
    for (int q = 0; q < K; ++q) { const float4 x = __ldg(src + q); f[4 * q] = x.x; f[4 * q + 1] = x.y; f[4 * q + 2] = x.z; f[4 * q + 3] = x.w; }
#pragma unroll
    for (int kp = 0; kp < KP; ++kp)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float lo = f[c * K + 2 * kp], hi = 2 * kp + 1 < K ? f[c * K + 2 * kp + 1] : (BIAS_COL ? bvc[c] : 0.f);
        asm("mov.b64 %0, {%1, %2};" : "=l"(w[kp][c]) : "f"(lo), "f"(hi));
      }
  }
  unsigned long long b2[4];
  asm("mov.b64 %0, {%1, %2};" : "=l"(b2[0]) : "f"(bv.x), "f"(0.f));
  asm("mov.b64 %0, {%1, %2};" : "=l"(b2[1]) : "f"(bv.y), "f"(0.f));
  asm("mov.b64 %0, {%1, %2};" : "=l"(b2[2]) : "f"(bv.z), "f"(0.f));
  asm("mov.b64 %0, {%1, %2};" : "=l"(b2[3]) : "f"(bv.w), "f"(0.f));
  float* __restrict__ C = p.C + (int64_t)g * p.c_gs + (int64_t)m_base * p.ldc + n;
  __syncthreads();
  // rows r and r + 4: outputs in o0 / o1 (also stored), returns the two sign nibbles {row r | row r + 4 << 4}
  auto two_rows = [&](int r) -> uint32_t {
    unsigned long long a0[2 * KQ], a1[2 * KQ];
#pragma unroll
    for (int q = 0; q < KQ; ++q) {
      const ulonglong2 x0 = *reinterpret_cast<const ulonglong2*>(&As[r * LDS_A + 4 * q]);        // warp-uniform address: broadcast
      const ulonglong2 x1 = *reinterpret_cast<const ulonglong2*>(&As[(r + 4) * LDS_A + 4 * q]);
      a0[2 * q] = x0.x; a0[2 * q + 1] = x0.y; a1[2 * q] = x1.x; a1[2 * q + 1] = x1.y;
    }
    unsigned long long acc0[4], acc1[4];  // {bias + even-k partial, odd-k partial}
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      acc0[c] = BIAS_COL ? fl_mul2(a0[0], w[0][c]) : fl_fma2(a0[0], w[0][c], b2[c]);
      acc1[c] = BIAS_COL ? fl_mul2(a1[0], w[0][c]) : fl_fma2(a1[0], w[0][c], b2[c]);
    }
#pragma unroll
    for (int kp = 1; kp < KP; ++kp)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        acc0[c] = fl_fma2(a0[kp], w[kp][c], acc0[c]);
        acc1[c] = fl_fma2(a1[kp], w[kp][c], acc1[c]);
      }
    float o0[4], o1[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float e, o;
      asm("mov.b64 {%0, %1}, %2;" : "=f"(e), "=f"(o) : "l"(acc0[c]));
      o0[c] = fmaxf(e + o, 0.f);
      asm("mov.b64 {%0, %1}, %2;" : "=f"(e), "=f"(o) : "l"(acc1[c]));
      o1[c] = fmaxf(e + o, 0.f);
    }
    *reinterpret_cast<float4*>(C + (int64_t)r * p.ldc) = make_float4(o0[0], o0[1], o0[2], o0[3]);
    *reinterpret_cast<float4*>(C + (int64_t)(r + 4) * p.ldc) = make_float4(o1[0], o1[1], o1[2], o1[3]);
    if (!BITS) return 0u;
    return (o0[0] > 0.f ? 1u : 0u) | (o0[1] > 0.f ? 2u : 0u) | (o0[2] > 0.f ? 4u : 0u) | (o0[3] > 0.f ? 8u : 0u) | (o1[0] > 0.f ? 16u : 0u) | (o1[1] > 0.f ? 32u : 0u) |
           (o1[2] > 0.f ? 64u : 0u) | (o1[3] > 0.f ? 128u : 0u);
  };
  if (!BITS) {
    for (int r = tr; r < rows; r += 8) two_rows(r);  // rows is a multiple of 8
    return;
  }
  // Sign-bit words for the backward mask (word = 32 columns = the nibbles of 8 consecutive lanes). The nibbles of 8 rows are collected in one register
  // (nibble i <-> row rb + 8 (i / 2) + 4 (i % 2)) and an 8 x 8 nibble transpose over the 8 lanes (3 butterfly steps, one shuffle each) leaves lane l with
  // the complete word of row i = l: 3 shuffles per 8 rows instead of 3 per row. rows % 32 == 0 (launch condition).
  const int l = tid & 7;
  for (int rb = tr; rb < rows; rb += 32) {
    uint32_t V = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) V |= two_rows(rb + 8 * q) << (8 * q);
#pragma unroll
    for (int d = 4; d >= 1; d >>= 1) {
      const uint32_t md = d == 4 ? 0xFFFF0000u : (d == 2 ? 0xFF00FF00u : 0xF0F0F0F0u);  // nibbles whose index has bit d set
      const bool hi = (l & d) != 0;
      const uint32_t send = hi ? (V & ~md) << (4 * d) : (V & md) >> (4 * d);
      const uint32_t recv = __shfl_xor_sync(0xffffffffu, send, d);
      V = (hi ? (V & md) : (V & ~md)) | recv;
    }
    const int row = rb + 8 * (l >> 1) + 4 * (l & 1);
    p.bits_out[(int64_t)g * p.bits_out_gs + (int64_t)(m_base + row) * 8 + ((tid & 63) >> 3)] = V;
  }
}

bool first_layer_reg_eligible(const GemmArgs& a) {
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  const bool k_ok = a.K == 11 || a.K == 12 || a.K == 14 || a.K == 15 || a.K == 16;  // hopper-sized inputs (state 11 (+1 absorbing), + 3 action columns)
  return k_ok && a.N == 256 && a.M % 8 == 0 && a.ldb == a.K && al16(a.B) && a.b_gs % 4 == 0;
}

template <int K>
static int launch_first_layer_reg(il_handle* h, const GemmArgs& a, cudaStream_t stream) {
  if (a.bits_out) IL_LAUNCH(h, (first_layer_reg_kernel<K, true>), dim3((a.M + 255) / 256, a.G), 256, 0, stream, a);
  else IL_LAUNCH(h, (first_layer_reg_kernel<K, false>), dim3((a.M + 255) / 256, a.G), 256, 0, stream, a);
  return 0;
}

bool first_layer_eligible(const GemmArgs& a) {
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  return a.a_kmajor && a.b_kmajor && a.K <= FL_K && a.N % FL_COLS == 0 && a.M % FL_ROWS == 0 && a.act == IL_ACT_RELU && a.bias && !a.mask && !a.colsum && !a.accumulate &&
         al16(a.C) && a.ldc % 4 == 0 && a.c_gs % 4 == 0 && al16(a.bias) && a.bias_gs % 4 == 0;
}

bool thin_k_eligible(const GemmArgs& a) {
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (a.K > TK_MAXK || !a.a_kmajor || a.N < 64 || a.N % 4 || a.colsum || a.accumulate) return false;
  if (!al16(a.C) || a.ldc % 4 || a.c_gs % 4) return false;
  if (a.bias && (!al16(a.bias) || a.bias_gs % 4)) return false;
  if (a.mask && (!al16(a.mask) || a.ldmask % 4 || a.mask_gs % 4)) return false;
  return true;
}

// Streaming kernels for head-shaped products whose cost is one pass over a [K, wide] or [M, wide] activation matrix
// (wide = hidden width) while the other operand and the output are tiny (<= 16 columns). HBM-bound by construction.
constexpr int ST_MAXS = 16;
// TN: C[m][n] = sum_k A[k][m] * B[k][n] (A stored [K, M], B stored [K, N]) with min(M, N) <= 16. WIDE_A: M is the wide side
// (first-layer weight gradient: A = dZ [B, H], B = X [B, S]); else N is wide (last-layer weight gradient: A = dOut [B, NH],
// B = H2 [B, H]). One CTA per (group, 256 wide columns); each thread owns one wide column and streams it over K.
template <bool WIDE_A>
__global__ void __launch_bounds__(256) gemm_stream_tn_kernel(const GemmArgs p) {
  extern __shared__ __align__(16) float U[];  // [K][ST_MAXS] small operand, zero padded
  const int g = blockIdx.y, w0 = blockIdx.x * 256, tid = threadIdx.x;
  const int K = p.K, S = WIDE_A ? p.N : p.M, W = WIDE_A ? p.M : p.N;
  const float* __restrict__ A = p.A + (int64_t)(g / p.a_gdiv) * p.a_gs;
  const float* __restrict__ B = p.B + (int64_t)(g / p.b_gdiv) * p.b_gs;
  const float* __restrict__ T = WIDE_A ? A : B;
  const float* __restrict__ Us = WIDE_A ? B : A;
  const int ldt = WIDE_A ? p.lda : p.ldb, ldu = WIDE_A ? p.ldb : p.lda;
  for (int idx = tid; idx < K * ST_MAXS; idx += 256) {
    const int k = idx / ST_MAXS, j = idx % ST_MAXS;
    U[idx] = j < S ? __ldg(Us + (int64_t)k * ldu + j) : 0.f;
  }
  __syncthreads();
  const int w = w0 + tid;
  float acc[ST_MAXS], tsum = 0.f;
#pragma unroll
  for (int j = 0; j < ST_MAXS; ++j) acc[j] = 0.f;
  if (w < W) {
    const float* tp = T + w;
    int k = 0;
    float tn[8];  // software pipeline: the next 8 rows are in flight while the current 8 are consumed (the loop is latency-bound)
    if (K >= 8) {
#pragma unroll
      for (int u = 0; u < 8; ++u) tn[u] = __ldg(tp + (int64_t)u * ldt);
    }
    for (; k + 8 <= K; k += 8) {
      float t[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) t[u] = tn[u];
      if (k + 16 <= K) {
#pragma unroll
        for (int u = 0; u < 8; ++u) tn[u] = __ldg(tp + (int64_t)(k + 8 + u) * ldt);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        tsum += t[u];
        const float4* ur = reinterpret_cast<const float4*>(U + (k + u) * ST_MAXS);
#pragma unroll
        for (int q = 0; q < ST_MAXS / 4; ++q) {
          if (q * 4 < S) {
            const float4 uv = ur[q];
            acc[q * 4 + 0] = fmaf(t[u], uv.x, acc[q * 4 + 0]); acc[q * 4 + 1] = fmaf(t[u], uv.y, acc[q * 4 + 1]);
            acc[q * 4 + 2] = fmaf(t[u], uv.z, acc[q * 4 + 2]); acc[q * 4 + 3] = fmaf(t[u], uv.w, acc[q * 4 + 3]);
          }
        }
      }
    }
    for (; k < K; ++k) {
      const float t = __ldg(tp + (int64_t)k * ldt);
      tsum += t;
#pragma unroll
      for (int j = 0; j < ST_MAXS; ++j) acc[j] = fmaf(t, U[k * ST_MAXS + j], acc[j]);
    }
    float* __restrict__ C = p.C + (int64_t)g * p.c_gs;
    if (WIDE_A) {  // C[m = w][n = j]
#pragma unroll
      for (int j = 0; j < ST_MAXS; ++j)
        if (j < S) C[(int64_t)w * p.ldc + j] = acc[j];
      if (p.colsum) p.colsum[(int64_t)g * p.colsum_gs + w] = tsum;  // sum_k A[k][m]
    } else {       // C[m = j][n = w]
#pragma unroll
      for (int j = 0; j < ST_MAXS; ++j)
        if (j < S) C[(int64_t)j * p.ldc + w] = acc[j];
    }
  }
  if (!WIDE_A && p.colsum && blockIdx.x == 0 && tid < S) {  // sum_k A[k][m] of the small operand
    float s = 0.f;
    for (int k = 0; k < K; ++k) s += U[k * ST_MAXS + tid];
    p.colsum[(int64_t)g * p.colsum_gs + tid] = s;
  }
}


// First-layer weight gradient, specialised: C[m][j] = sum_k A[k][m] * B[k][j] (+ colsum[m] = sum_k A[k][m]) with A = dZ [K = batch rows, M = hidden
// columns] wide and B = X [K, N <= 16 input columns] narrow. One CTA per (net, 256 hidden columns): 64 column-threads (a 128-bit slice of every
// dZ row each) x 4 row groups, 4 rows in flight per thread, the narrow operand broadcast from shared memory; the row groups are combined through
// shared memory in a fixed order. (The streaming kernel above walks one column per thread with 8 scalar loads in flight: 2.1 TB/s.)
constexpr int WT_MAXN = 16;
__global__ void __launch_bounds__(256, 2) wide_tn_kernel(const GemmArgs p) {
  extern __shared__ __align__(16) float wt_sm[];  // X [K][WT_MAXN] zero padded, then the reduction scratch [4][WT_MAXN + 1][64] float4
  const int g = blockIdx.y, tid = threadIdx.x, tc = tid & 63, tr = tid >> 6, col = blockIdx.x * 256 + tc * 4, K = p.K, N = p.N;
  float* xs = wt_sm;
  float4* red = reinterpret_cast<float4*>(wt_sm + K * WT_MAXN);
  const float* __restrict__ A = p.A + (int64_t)(g / p.a_gdiv) * p.a_gs;
  const float* __restrict__ B = p.B + (int64_t)(g / p.b_gdiv) * p.b_gs;
  const bool active = col < p.M;
  const float* ap = A + col;
  float4 d[4], dn[4];
  auto fetch = [&](float4 (&dst)[4], int k0) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int k = k0 + 4 * u;
      dst[u] = (active && k < K) ? __ldg(reinterpret_cast<const float4*>(ap + (int64_t)k * p.lda)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  fetch(d, tr);  // the first wide rows are in flight while the small operand is staged
  for (int i = tid; i < K * WT_MAXN; i += 256) {
    const int k = i / WT_MAXN, j = i % WT_MAXN;
    xs[i] = j < N ? __ldg(B + (int64_t)k * p.ldb + j) : 0.f;
  }
  __syncthreads();
  float4 acc[WT_MAXN], cs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int j = 0; j < WT_MAXN; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (active) {
    for (int k0 = tr; k0 < K; k0 += 16) {
      fetch(dn, k0 + 16);  // the next 4 rows are in flight while these 4 are consumed
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int k = k0 + 4 * u;
        if (k >= K) continue;
        cs.x += d[u].x; cs.y += d[u].y; cs.z += d[u].z; cs.w += d[u].w;
        // the whole (zero padded) row of the small operand first — four independent broadcast loads — then the FMAs: with one load in front of each
        // group of 16 FMAs the warp stalled on the shared-memory scoreboard four times per row
        float4 xv[WT_MAXN / 4];
#pragma unroll
        for (int q = 0; q < WT_MAXN / 4; ++q) xv[q] = *reinterpret_cast<const float4*>(xs + k * WT_MAXN + 4 * q);
#pragma unroll
        for (int q = 0; q < WT_MAXN / 4; ++q) {
          if (q * 4 < N) {
            const float xj[4] = {xv[q].x, xv[q].y, xv[q].z, xv[q].w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              float4& a = acc[q * 4 + e];
              a.x = fmaf(d[u].x, xj[e], a.x); a.y = fmaf(d[u].y, xj[e], a.y); a.z = fmaf(d[u].z, xj[e], a.z); a.w = fmaf(d[u].w, xj[e], a.w);
            }
          }
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) d[u] = dn[u];
    }
  }
#pragma unroll
  for (int j = 0; j < WT_MAXN; ++j) red[(tr * (WT_MAXN + 1) + j) * 64 + tc] = acc[j];
  red[(tr * (WT_MAXN + 1) + WT_MAXN) * 64 + tc] = cs;
  __syncthreads();
  if (active) {  // every row group finishes a quarter of the outputs (fixed summation order over the 4 partials)
    float* __restrict__ C = p.C + (int64_t)g * p.c_gs;
#pragma unroll
    for (int jj = 0; jj < (WT_MAXN + 4) / 4; ++jj) {
      const int j = tr + 4 * jj;
      if (j > WT_MAXN) continue;
      if (j < N || j == WT_MAXN) {
        float4 a = red[(0 * (WT_MAXN + 1) + j) * 64 + tc];
#pragma unroll
        for (int q = 1; q < 4; ++q) {
          const float4 t = red[(q * (WT_MAXN + 1) + j) * 64 + tc];
          a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
        }
        if (j == WT_MAXN) {
          if (p.colsum) *reinterpret_cast<float4*>(p.colsum + (int64_t)g * p.colsum_gs + col) = a;
        } else {
          C[(int64_t)(col + 0) * p.ldc + j] = a.x; C[(int64_t)(col + 1) * p.ldc + j] = a.y; C[(int64_t)(col + 2) * p.ldc + j] = a.z; C[(int64_t)(col + 3) * p.ldc + j] = a.w;
        }
      }
    }
  }
}
bool wide_tn_eligible(const GemmArgs& a) {
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  return !a.a_kmajor && !a.b_kmajor && a.N <= WT_MAXN && a.M >= 64 && a.M % 4 == 0 && a.K <= 1024 && !a.bias && a.act < 0 && !a.mask && !a.accumulate && al16(a.A) && a.lda % 4 == 0 &&
         a.a_gs % 4 == 0 && (!a.colsum || (al16(a.colsum) && a.colsum_gs % 4 == 0));
}


// First-layer input gradient, specialised: C[m][j] = sum_k A[m][k] * B[k][j] with A = dZ [M = batch rows, K = hidden width, K-major] and a narrow
// B = a column slice of W_1 [K, N <= 8] (the action columns, training.py:36-41). One warp per row: the lanes own 4-wide slices of k (128-bit
// coalesced loads of the row), their slice of B lives in registers for the whole CTA, 4 rows in flight, butterfly reduction per row.
constexpr int RD_MAXN = 8, RD_MAXKV = 4;  // N <= 8 output columns, K <= 512 (K / 128 float4 per lane)
constexpr int RD_ROWS = 256;              // rows per CTA: the register-resident slice of B is loaded once per 256 rows (was 64: the strided prologue dominated the CTA's life)
template <int RD_MAXKV, int RD_MAXN>
__global__ void __launch_bounds__(256) row_dot_kernel(const GemmArgs p) {
  const int g = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, N = p.N, kv = p.K / 128;
  const float* __restrict__ A = p.A + (int64_t)(g / p.a_gdiv) * p.a_gs;
  const float* __restrict__ B = p.B + (int64_t)(g / p.b_gdiv) * p.b_gs;
  float w[RD_MAXKV][4][RD_MAXN];  // this lane's k values x output columns
#pragma unroll
  for (int v = 0; v < RD_MAXKV; ++v)
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
      for (int j = 0; j < RD_MAXN; ++j) w[v][e][j] = (v < kv && j < N) ? __ldg(B + (int64_t)(v * 128 + lane * 4 + e) * p.ldb + j) : 0.f;
  float* __restrict__ C = p.C + (int64_t)g * p.c_gs;
  const int m_end = min(p.M, (int)(blockIdx.x + 1) * RD_ROWS);
  constexpr bool PF = RD_MAXKV <= 2;  // the prefetch buffer does not fit next to a K = 512 slice of B
  float4 a[4][RD_MAXKV], an[PF ? 4 : 1][RD_MAXKV];
  auto fetch = [&](float4 (*dst)[RD_MAXKV], int m0) {  // rows m0, m0 + 8, m0 + 16, m0 + 24
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < RD_MAXKV; ++v) {
        const int m = m0 + 8 * u;
        dst[u][v] = (v < kv && m < m_end) ? __ldg(reinterpret_cast<const float4*>(A + (int64_t)m * p.lda + v * 128 + lane * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
  };
  fetch(a, blockIdx.x * RD_ROWS + warp);
  for (int m0 = blockIdx.x * RD_ROWS + warp; m0 < m_end; m0 += 32) {
    if (PF) fetch(an, m0 + 32);  // the next 4 rows of this warp are in flight while these 4 are reduced
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int m = m0 + 8 * u;
      float acc[RD_MAXN];
#pragma unroll
      for (int j = 0; j < RD_MAXN; ++j) {
        float t = 0.f;
#pragma unroll
        for (int v = 0; v < RD_MAXKV; ++v) t = fmaf(a[u][v].x, w[v][0][j], fmaf(a[u][v].y, w[v][1][j], fmaf(a[u][v].z, w[v][2][j], fmaf(a[u][v].w, w[v][3][j], t))));
        acc[j] = t;
      }
#pragma unroll
      for (int j = 0; j < RD_MAXN; ++j)
        if (j < N) acc[j] = warp_sum(acc[j]);
      if (m < m_end && lane < N) {
        float v = acc[0];
#pragma unroll
        for (int j = 1; j < RD_MAXN; ++j) v = lane == j ? acc[j] : v;
        C[(int64_t)m * p.ldc + lane] = v;
      }
    }
    if (PF) {
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < RD_MAXKV; ++v) a[u][v] = an[PF ? u : 0][v];
    } else if (m0 + 32 < m_end) {
      fetch(a, m0 + 32);
    }
  }
}
bool row_dot_eligible(const GemmArgs& a) {
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  return a.a_kmajor && !a.b_kmajor && a.N <= RD_MAXN && a.K % 128 == 0 && a.K <= 128 * RD_MAXKV && a.M >= 32 && !a.bias && a.act < 0 && !a.mask && !a.accumulate && !a.colsum &&
         al16(a.A) && a.lda % 4 == 0 && a.a_gs % 4 == 0;
}

template <int BM, int BN, int TM, int TN>
int launch_cfg(il_handle* h, const GemmArgs& a, cudaStream_t stream) {
  constexpr int BK = 16;
  dim3 grid((a.N + BN - 1) / BN, (a.M + BM - 1) / BM, a.G), block(256);
  if (a.a_kmajor && a.b_kmajor) {
    IL_LAUNCH(h, (gemm_grouped_kernel<BM, BN, BK, TM, TN, true, true>), grid, block, 0, stream, a);
  } else if (a.a_kmajor && !a.b_kmajor) {
    IL_LAUNCH(h, (gemm_grouped_kernel<BM, BN, BK, TM, TN, true, false>), grid, block, 0, stream, a);
  } else if (!a.a_kmajor && !a.b_kmajor) {
    IL_LAUNCH(h, (gemm_grouped_kernel<BM, BN, BK, TM, TN, false, false>), grid, block, 0, stream, a);
  } else {
    IL_FAIL("gemm: unsupported operand layout (A m-major with B k-major)");
  }
  return 0;
}

}  // namespace

bool gemm_uses_tc(const il_handle* h, const GemmArgs& a) {
  return a.M >= 128 && a.N >= 128 && a.K >= 128 && h->gemm_mode != IL_GEMM_FP32 && tc_gemm_eligible(a);
}
// launch_gemm routes this first-layer shape to first_layer_reg_kernel, which can also emit the ReLU sign-bit words
bool gemm_first_layer_emits_bits(const il_handle* h, const GemmArgs& a) {
  return h->first_layer_fast >= 2 && a.M > 16 && a.M % 32 == 0 && first_layer_eligible(a) && first_layer_reg_eligible(a);
}

int gemm_init() {
  IL_CUDA(cudaFuncSetAttribute(wide_tn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (1024 * WT_MAXN + 4 * (WT_MAXN + 1) * 64 * 4) * 4));
  IL_CUDA(cudaFuncSetAttribute(gemm_stream_tn_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  IL_CUDA(cudaFuncSetAttribute(gemm_stream_tn_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  return 0;
}

// Compulsory HBM traffic of one grouped GEMM: every distinct operand element read once, every output written once.
double gemm_algorithmic_bytes(const GemmArgs& a, bool stores_c) {
  const double ga = (a.G + a.a_gdiv - 1) / a.a_gdiv, gb = (a.G + a.b_gdiv - 1) / a.b_gdiv;
  double b = 4.0 * (ga * a.M * a.K + gb * a.K * a.N);
  if (stores_c) b += 4.0 * a.G * (double)a.M * a.N;
  if (a.mask_bits) b += 4.0 * a.G * (double)a.M * (a.N / 32);
  else if (a.mask) b += 4.0 * a.G * (double)a.M * a.N;
  if (a.bias) b += 4.0 * a.G * a.N;
  return b;
}
int profile_open(il_handle* h, ProfiledLaunch* pl, double flops, double bytes, cudaStream_t stream) {
  IL_CUDA(cudaEventCreate(&pl->start));
  IL_CUDA(cudaEventCreate(&pl->stop));
  pl->flops = flops;
  pl->bytes = bytes;
  IL_CUDA(cudaEventRecord(pl->start, stream));
  return 0;
}
int profile_close(il_handle* h, ProfiledLaunch* pl, cudaStream_t stream) {
  IL_CUDA(cudaEventRecord(pl->stop, stream));
  h->profiled.push_back(*pl);
  return 0;
}

int launch_gemm(il_handle* h, const GemmArgs& a, cudaStream_t stream) {
  IL_CHECK(a.M > 0 && a.N > 0 && a.K > 0 && a.G > 0, "gemm: empty problem M=%d N=%d K=%d G=%d", a.M, a.N, a.K, a.G);
  IL_CHECK(a.G <= 65535, "gemm: too many groups (%d)", a.G);
  IL_CHECK(!(a.colsum && a.a_kmajor), "gemm: colsum needs the [K, M] operand layout");
  IL_CHECK(!(a.accumulate && a.act >= 0), "gemm: accumulate with activation is not supported");
  const bool plain = !a.bias && a.act < 0 && !a.mask && !a.mask_bits && !a.accumulate;
  IL_CHECK(!a.mask_bits || gemm_uses_tc(h, a), "gemm: sign-bit masks need the wgmma engine (M=%d N=%d K=%d)", a.M, a.N, a.K);
  IL_CHECK(!a.bits_out || gemm_first_layer_emits_bits(h, a), "gemm: this launch cannot emit sign-bit words (M=%d N=%d K=%d)", a.M, a.N, a.K);
  if (h->wide_tn && row_dot_eligible(a)) {
    const dim3 grid((a.M + RD_ROWS - 1) / RD_ROWS, a.G);
    if (a.K <= 256 && a.N <= 4) IL_LAUNCH(h, (row_dot_kernel<2, 4>), grid, 256, 0, stream, a);
    else if (a.K <= 256) IL_LAUNCH(h, (row_dot_kernel<2, 8>), grid, 256, 0, stream, a);
    else IL_LAUNCH(h, (row_dot_kernel<4, 8>), grid, 256, 0, stream, a);
    return 0;
  }
  if (h->wide_tn && a.K >= 64 && wide_tn_eligible(a)) {
    const size_t smem = ((size_t)a.K * WT_MAXN + 4 * (WT_MAXN + 1) * 64 * 4) * sizeof(float);
    IL_LAUNCH(h, wide_tn_kernel, dim3((a.M + 255) / 256, a.G), 256, smem, stream, a);
    return 0;
  }
  if (plain && !a.a_kmajor && !a.b_kmajor && a.K >= 64 && a.K * ST_MAXS * 4 <= 64 * 1024 && ((a.M <= ST_MAXS && a.N >= 64) || (a.N <= ST_MAXS && a.M >= 64))) {
    const bool wide_a = a.N <= ST_MAXS && a.M >= 64;
    const int W = wide_a ? a.M : a.N;
    dim3 grid((W + 255) / 256, a.G);
    const size_t smem = (size_t)a.K * ST_MAXS * 4;
    if (wide_a) IL_LAUNCH(h, gemm_stream_tn_kernel<true>, grid, 256, smem, stream, a);
    else IL_LAUNCH(h, gemm_stream_tn_kernel<false>, grid, 256, smem, stream, a);
    return 0;
  }
  if (h->first_layer_fast >= 2 && a.M > 16 && first_layer_eligible(a) && first_layer_reg_eligible(a)) {
    switch (a.K) {
      case 11: return launch_first_layer_reg<11>(h, a, stream);
      case 12: return launch_first_layer_reg<12>(h, a, stream);
      case 14: return launch_first_layer_reg<14>(h, a, stream);
      case 15: return launch_first_layer_reg<15>(h, a, stream);
      default: return launch_first_layer_reg<16>(h, a, stream);
    }
  }
  if (h->first_layer_fast && a.M > 16 && first_layer_eligible(a)) {
    dim3 grid(a.N / FL_COLS, (a.M + FL_ROWS * FL_ITERS - 1) / (FL_ROWS * FL_ITERS), a.G);
    IL_LAUNCH(h, first_layer_relu_kernel, grid, 256, 0, stream, a);
    return 0;
  }
  if (a.M > 16 && thin_k_eligible(a)) {
    dim3 grid((a.N + TK_COLS - 1) / TK_COLS, (a.M + TK_ROWS * TK_ITERS - 1) / (TK_ROWS * TK_ITERS), a.G);
    if (a.mask && h->thin_hoist) {
      if (a.b_kmajor) IL_LAUNCH(h, (gemm_thin_k_kernel<true, true>), grid, 256, 0, stream, a);
      else IL_LAUNCH(h, (gemm_thin_k_kernel<false, true>), grid, 256, 0, stream, a);
      return 0;
    }
    if (a.b_kmajor) IL_LAUNCH(h, (gemm_thin_k_kernel<true, false>), grid, 256, 0, stream, a);
    else IL_LAUNCH(h, (gemm_thin_k_kernel<false, false>), grid, 256, 0, stream, a);
    return 0;
  }
  if (a.M <= 16) return launch_cfg<16, 128, 1, 8>(h, a, stream);
  if (a.N <= 16) return launch_cfg<128, 16, 8, 1>(h, a, stream);
  if (a.M <= 32) return launch_cfg<32, 128, 2, 8>(h, a, stream);
  const bool dense = a.M >= 128 && a.N >= 128 && a.K >= 128;  // the H x H hidden-layer contractions (SURVEY §8d)
  const bool tc = gemm_uses_tc(h, a);
  auto run = [&]() { return tc ? launch_tc_gemm(h, a, stream) : launch_cfg<128, 128, 8, 8>(h, a, stream); };
  if (h->profiling && dense) {
    ProfiledLaunch pl;
    IL_TRY(profile_open(h, &pl, 2.0 * a.M * a.N * a.K * a.G, gemm_algorithmic_bytes(a, true), stream));
    const int rc = run();
    IL_TRY(profile_close(h, &pl, stream));
    return rc;
  }
  return run();
}

// Test / diagnostics entry: one grouped GEMM with the fused epilogues, routed like the MLP programs route it.
extern "C" int il_debug_gemm(il_handle* h, int M, int N, int K, int G, const float* A, int64_t a_gs, int lda, int a_kmajor, const float* B, int64_t b_gs, int ldb, int b_kmajor,
                             float* C, int64_t c_gs, int ldc, const float* bias, int64_t bias_gs, int act, const float* mask, int64_t mask_gs, int ldmask, int mask_act,
                             float* colsum, int64_t colsum_gs, void* stream) {
  IL_CHECK(h && A && B && C, "il_debug_gemm: null argument");
  GemmArgs a{};
  a.A = A; a.a_gs = a_gs; a.a_gdiv = 1; a.lda = lda; a.a_kmajor = a_kmajor;
  a.B = B; a.b_gs = b_gs; a.b_gdiv = 1; a.ldb = ldb; a.b_kmajor = b_kmajor;
  a.C = C; a.c_gs = c_gs; a.ldc = ldc; a.bias = bias; a.bias_gs = bias_gs; a.act = act;
  a.mask = mask; a.mask_gs = mask_gs; a.ldmask = ldmask; a.mask_act = mask_act; a.colsum = colsum; a.colsum_gs = colsum_gs;
  a.M = M; a.N = N; a.K = K; a.G = G;
  return launch_gemm(h, a, (cudaStream_t)stream);
}

extern "C" int il_profile_begin(il_handle* h) {
  IL_CHECK(h, "il_profile_begin: null handle");
  h->profiled.clear();
  h->profiling = 1;
  return 0;
}

extern "C" int il_profile_end(il_handle* h, double* total_ms, double* total_flops, int64_t* launches) {
  IL_CHECK(h && total_ms && total_flops && launches, "il_profile_end: null argument");
  h->profiling = 0;
  IL_CUDA(cudaDeviceSynchronize());
  double ms = 0.0, fl = 0.0, by = 0.0;
  for (auto& pl : h->profiled) {
    float e = 0.f;
    IL_CUDA(cudaEventElapsedTime(&e, pl.start, pl.stop));
    ms += e;
    fl += pl.flops;
    by += pl.bytes;
    cudaEventDestroy(pl.start);
    cudaEventDestroy(pl.stop);
  }
  *total_ms = ms; *total_flops = fl; *launches = (int64_t)h->profiled.size();
  h->profiled_bytes = by;
  h->profiled.clear();
  return 0;
}

extern "C" int il_profile_bytes(il_handle* h, double* total_bytes) {
  IL_CHECK(h && total_bytes, "il_profile_bytes: null argument");
  *total_bytes = h->profiled_bytes;
  return 0;
}
