// Shared device/host helpers for the sm_90a hot path. Compiled only for sm_90a (see build.py).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <vector>

#include "../../include/il_b200.h"

#define IL_MAX_GRID_Y 65535  // the per-replica RNG launches put the replica on gridDim.y

struct ProfiledLaunch {
  cudaEvent_t start, stop;
  double flops;
  double bytes;   // algorithmic (compulsory) HBM bytes of the launch: unique operand bytes read + output bytes written
};
struct il_handle {
  int device;
  int sm_count;
  int gemm_mode;
  int thin_hoist;                       // K-thin kernel: hoisted mask loads for the masked (dX) variant (IL_THIN_HOIST=0/1)
  int wide_tn;                          // first-layer weight gradient: 128-bit row-group kernel (IL_WIDE_TN=0 keeps the column-streaming kernel)
  int first_layer_fast;                 // first MLP layer: specialised k-pair FFMA kernel for K <= 16 (IL_FIRST_LAYER_FAST=0 keeps the generic K-thin kernel)
  int mask_bits;                        // ReLU masks of the MLP backward as sign-bit words written by the forward kernels (IL_MASK_BITS=0: fp32 activations as masks)
  int head_fused;                       // MLP backward: fused head kernel (dZ, dW_L, db_L, db_{L-1} in one pass; IL_HEAD_FUSED=0 disables)
  int debug_sync;                       // IL_DEBUG_SYNC=1: multi-kernel programs synchronise after every stage and name the one that failed
  int adam_tma;                         // AdamW: TMA-staged (cp.async.bulk) streaming kernel for large flat buffers (IL_ADAM_TMA=1 enables)
  int gail_tiled;                       // GAIL update: register-tiled kernel for d <= 32 (IL_GAIL_TILED=0 keeps the first kernel)
  int tc_fuse_l1;                       // wgmma engine: compute the first MLP layer in place of the A operand loads of the second (IL_TC_FUSE_L1=1 enables)
  long long launches;
  int profiling;                        // il_profile_begin/end: CUDA events around every dense-layer GEMM launch
  std::vector<ProfiledLaunch> profiled;
  double profiled_bytes;                // summed by the last il_profile_end
  void* eval_graph;                     // cached evaluation-rollout graph (eval.cu)
  cudaStream_t build_stream;            // private stream used only to CAPTURE graphs (the legacy default stream cannot capture)
};
void il_eval_release(il_handle* h);

extern thread_local char g_il_error[512];

#define IL_FAIL(...)                                     \
  do {                                                   \
    snprintf(g_il_error, sizeof(g_il_error), __VA_ARGS__); \
    return 1;                                            \
  } while (0)

#define IL_CHECK(cond, ...)        \
  do {                             \
    if (!(cond)) IL_FAIL(__VA_ARGS__); \
  } while (0)

#define IL_CUDA(expr)                                                                             \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) IL_FAIL("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// Launch + count + check (cudaPeekAtLastError is legal during stream capture).
#define IL_LAUNCH(h, kernel, grid, block, smem, stream, ...)                                      \
  do {                                                                                            \
    kernel<<<(grid), (block), (smem), (cudaStream_t)(stream)>>>(__VA_ARGS__);                     \
    (h)->launches++;                                                                              \
    cudaError_t _e = cudaPeekAtLastError();                                                       \
    if (_e != cudaSuccess) IL_FAIL("launch of %s failed: %s (%s:%d)", #kernel, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

#define IL_TRY(expr)          \
  do {                        \
    int _r = (expr);          \
    if (_r != 0) return _r;   \
  } while (0)

__host__ __device__ static inline int64_t il_align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// ---- row layout (il_batch / il_replay) -------------------------------------------------------------------
struct RowLayout {
  int state, action, reward, next_state, terminal, timeout, weight, step, len;
};
__host__ __device__ inline RowLayout row_layout(int S, int A) {
  RowLayout L;
  L.state = 0;
  L.action = S;
  L.reward = S + A;
  L.next_state = S + A + 1;
  L.terminal = 2 * S + A + 1;
  L.timeout = L.terminal + 1;
  L.weight = L.terminal + 2;
  L.step = L.terminal + 3;
  L.len = (2 * S + A + 5 + 3) / 4 * 4;
  return L;
}

// ---- MLP flat-parameter layout ---------------------------------------------------------------------------
struct MlpOffsets {
  int64_t w[IL_MAX_LAYERS], b[IL_MAX_LAYERS], total;
};
__host__ __device__ static inline MlpOffsets mlp_offsets(const int32_t* dims, int n_layers) {
  MlpOffsets o;
  int64_t off = 0;
  for (int l = 0; l < n_layers; ++l) {
    o.w[l] = off;
    off = il_align_up(off + (int64_t)dims[l + 1] * dims[l], 4);
    o.b[l] = off;
    off = il_align_up(off + dims[l + 1], 4);
  }
  o.total = il_align_up(off, 32);
  return o;
}

// ---- device math -------------------------------------------------------------------------------------------
__device__ __forceinline__ float act_apply(float x, int act) {
  if (act == IL_ACT_RELU) return fmaxf(x, 0.f);
  if (act == IL_ACT_TANH) return tanhf(x);
  return 1.f / (1.f + expf(-x));
}
// derivative of the activation expressed through its OUTPUT y
__device__ __forceinline__ float act_grad_from_output(float y, int act) {
  if (act == IL_ACT_RELU) return y > 0.f ? 1.f : 0.f;
  if (act == IL_ACT_TANH) return 1.f - y * y;
  return y * (1.f - y);
}
__device__ __forceinline__ float softplusf(float x) {  // torch softplus (beta 1, threshold 20)
  return x > 20.f ? x : log1pf(expf(x));
}
__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }

// ---- AdamW (torch _single_tensor_adam: Python-double scalars, then cast to the tensor dtype) ----------------------
struct AdamW {
  float step_size, bc2_sqrt;  // lr / (1 - beta1^t), sqrt(1 - beta2^t)
  float decay, w1, w2, beta2, eps;  // 1 - lr * wd (one rounding: the fused multiply-add the expression always compiled to), 1 - beta1, 1 - beta2
  bool has_wd;
};
// the two step-dependent scalars, computed by one thread and staged by the caller (shared memory or registers)
__device__ __forceinline__ void adamw_bias_correction(double lr, double beta1, double beta2, int64_t step, float& step_size, float& bc2_sqrt) {
  const double t = (double)step;
  step_size = (float)(lr / (1.0 - pow(beta1, t)));
  bc2_sqrt = (float)sqrt(1.0 - pow(beta2, t));
}
__device__ __forceinline__ AdamW adamw_coefs(float step_size, float bc2_sqrt, double lr, double wd, double beta1, double beta2, double eps) {
  return AdamW{step_size, bc2_sqrt, (float)fma(-lr, wd, 1.0), (float)(1.0 - beta1), (float)(1.0 - beta2), (float)beta2, (float)eps, wd != 0.0};
}
// one element; step_size / decay / has_wd are passed separately so per-replica tables can override them
__device__ __forceinline__ void adamw_update(const AdamW& c, float& p, float& m, float& v, float g, float step_size, float decay, bool has_wd) {
  if (has_wd) p = __fmul_rn(p, decay);                                          // param.mul_(1 - lr * weight_decay)
  m = __fadd_rn(m, __fmul_rn(c.w1, __fsub_rn(g, m)));                           // exp_avg.lerp_(grad, 1 - beta1)
  v = __fadd_rn(__fmul_rn(v, c.beta2), __fmul_rn(__fmul_rn(c.w2, g), g));       // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
  const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), c.bc2_sqrt), c.eps);        // (exp_avg_sq.sqrt() / bias_correction2_sqrt).add_(eps)
  p = __fadd_rn(p, __fmul_rn(-step_size, __fdiv_rn(m, denom)));                 // param.addcdiv_(exp_avg, denom, value=-step_size)
}
__device__ __forceinline__ void adamw_update(const AdamW& c, float& p, float& m, float& v, float g) { adamw_update(c, p, m, v, g, c.step_size, c.decay, c.has_wd); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// Block-wide sum for blockDim.x <= 1024 (deterministic order); `red` is >= 32 floats of shared memory.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = 0.f;
  if (warp == 0) {
    r = lane < nw ? red[lane] : 0.f;
    r = warp_sum(r);
    if (lane == 0) red[0] = r;
  }
  __syncthreads();
  return red[0];
}

// ---- Philox4x32-10 ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    const uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}
__device__ __forceinline__ float u32_to_unit(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }  // [0, 1)

// ---- grouped GEMM (gemm.cu) ---------------------------------------------------------------------------------
// C[g] (M x N) = A[g] (M x K) * B[g] (K x N) with fused epilogue; all fp32.
struct GemmArgs {
  const float* A;        // a_kmajor: stored [M, K] (K contiguous, row stride lda); else stored [K, M] (M contiguous, row stride lda)
  int64_t a_gs;
  int a_gdiv, lda, a_kmajor;
  const float* B;        // b_kmajor: stored [N, K] (K contiguous, row stride ldb)  (a Linear weight); else stored [K, N] (N contiguous)
  int64_t b_gs;
  int b_gdiv, ldb, b_kmajor;
  float* C;              // [M, N], row stride ldc
  int64_t c_gs;
  int ldc;
  const float* bias;     // [N] per group or nullptr
  int64_t bias_gs;
  int act;               // -1 none, else IL_ACT_* applied to the output
  const float* mask;     // optional [M, N] (row stride ldmask): output *= act'(mask) with mask = activation OUTPUT
  int64_t mask_gs;
  int ldmask, mask_act;
  float* colsum;         // optional (only with !a_kmajor): colsum[m] = sum_k A[k, m]  (bias gradient)
  int64_t colsum_gs;
  int accumulate;        // C += result (before activation; only with act == -1)
  int M, N, K, G;
  // ReLU sign bits instead of fp32 activations where only the derivative mask is needed (1/32 of the bytes): word [m][n / 32], bit n % 32 set <=> output (m, n) > 0
  const uint32_t* mask_bits;  // alternative to `mask` (mask_act == relu); honoured by the wgmma engine
  int64_t mask_bits_gs;       // words per group
  uint32_t* bits_out;         // optional extra output of the kernels that support it (first_layer_reg_kernel, the fused-head wgmma launch)
  int64_t bits_out_gs;
};
int launch_gemm(il_handle* h, const GemmArgs& a, cudaStream_t stream);
bool gemm_uses_tc(const il_handle* h, const GemmArgs& a);                  // the dense wgmma engine takes this launch
bool gemm_first_layer_emits_bits(const il_handle* h, const GemmArgs& a);   // first_layer_reg_kernel takes this launch (bits_out supported)
double gemm_algorithmic_bytes(const GemmArgs& a, bool stores_c);
int profile_open(il_handle* h, ProfiledLaunch* pl, double flops, double bytes, cudaStream_t stream);
int profile_close(il_handle* h, ProfiledLaunch* pl, cudaStream_t stream);

// wgmma engine (tc_gemm.cu): dense M%128==0, N==256, K%16==0 problems when il_set_gemm_mode != IL_GEMM_FP32
bool tc_gemm_eligible(const GemmArgs& a);
int launch_tc_gemm(il_handle* h, const GemmArgs& a, cudaStream_t stream);
int tc_gemm_init();
// First MLP layer fused into the operand staging of the wgmma engine: the A operand of the dense product is
// relu(X W1^T + b1) (K0 = x_k <= 16 input columns), computed chunk by chunk into the operand tile instead of being read from HBM.
struct TcFuseL1 {
  const float* x;        // input rows: element (g, m, j) at x + (g / x_gdiv) * x_gs + m * x_ld + j
  int64_t x_gs;
  int x_gdiv, x_ld, x_k;
  const float* w1;       // [H, x_k] row-major per group (group stride gs), H = K of the dense product
  const float* b1;       // [H]
  int64_t gs;
  float* store;          // optional [G, M, H]: the first hidden activation, written when a backward pass needs it
  int64_t store_gs;
};
// dense hidden layer + bias + ReLU with the following (final, <= 8 units) linear layer fused into the epilogue
bool tc_head_fusable(const il_handle* h, const GemmArgs& a, int head_n);
bool tc_l1_fusable(const il_handle* h, const GemmArgs& a, int x_k);
bool tc_dx_head_fusable(const il_handle* h, const GemmArgs& a, int head_n);
int launch_tc_gemm_dx_head(il_handle* h, const GemmArgs& a, const float* w, int64_t w_gs, int w_ns, int head_n, float* out, int64_t out_gs, cudaStream_t stream);
int launch_tc_gemm_head(il_handle* h, const GemmArgs& a, const float* head_w, const float* head_b, int64_t head_gs, int head_n, float* head_out, int64_t head_out_gs, int store_c,
                        cudaStream_t stream, const TcFuseL1* l1 = nullptr);
