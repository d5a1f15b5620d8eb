// wgmma engine for the dense H x H layers of the replica-batched MLPs (sm_90a).
//
//   C[g] (M x N) = A[g] (M x K) * B[g] (K x N), fp32 in / fp32 out, tensor-core arithmetic:
//     IL_GEMM_TF32X3 : each operand is split x = hi + lo (hi = the top 19 bits of x, i.e. x truncated to tf32; lo = x - hi,
//                      exact in fp32) and the product is lo*hi + hi*lo + hi*hi with fp32 accumulation — fp32-level
//                      accuracy (error ~2^-21 per product, the dropped lo*lo term) at 3 MMAs per product ("3xTF32").
//     IL_GEMM_TF32   : hi*hi only (10-bit mantissa operands).
//
// Structure: persistent CTAs, one per SM, each walking the 128 x 256 output tiles blockIdx.x, blockIdx.x + gridDim.x, ...
// (the two M-tiles of a group run in the same wave, so the second read of B hits L2). The CTA is warp-specialised:
//   - warpgroup 0, the producer (56 registers per thread after setmaxnreg.dec; 72 with FUSE), copies A and B and splits B;
//   - warpgroups 1 and 2, the consumers (224 registers after setmaxnreg.inc; 216 with FUSE), split their A in registers,
//     multiply and run the epilogue. Consumer w owns rows [64 w, 64 w + 64) of the tile as the 128 fp32 accumulator
//     registers per thread of wgmma.mma_async m64n256k8.tf32.
// wgmma reads B from shared memory in K-major layout only and A either from there or from registers, and every operand
// needs the hi/lo split (a CUDA-core pass) anyway. Each A row is read by one consumer warpgroup only, so the consumers
// split A in their own registers and only B goes through shared-memory hi/lo tiles. Each k-block (16 floats of k) of the
// CTA's k-block stream (which runs on across tile boundaries) goes through three steps, all running at once on
// different k-blocks:
//   1. copy (producer): cp.async 16-byte copies of the raw fp32 chunks global -> shared memory, no registers held. B
//      goes to a RAW_STAGES-deep raw ring; each producer thread reads back exactly the B chunks it copied, so
//      cp.async.wait_group is all the visibility that ring needs (no TMA, which could not feed the tensor core anyway
//      because the split has to see every element). A goes straight to an A_STAGES-deep ring in the layout the
//      consumers read (see A_STAGES); with FUSE the producer computes the A chunks (the first MLP layer) into it instead;
//   2. split (producer): B's hi and lo tiles go into one of three hi/lo stages in the canonical K-major SWIZZLE_64B
//      layout. A B stored [K, rows] in global memory is transposed on the way: a thread splits a 4 (k) x 4 (rows) block
//      and stores four 16-byte k-chunks, in a per-thread rotated order that keeps the shared-memory stores conflict-free;
//   3. multiply (consumers): each consumer warpgroup loads the raw A fragments of its rows (ldmatrix or 32-bit loads,
//      conflict-free), splits them in registers and issues the 6 (3xTF32) or 2 (TF32) wgmmas of the k-block, A from
//      registers and B from the stage. The products, their hi/lo values and their order are the same as with both
//      operands in shared memory, so the results are too, bit for bit.
// The stages hand over through full / empty mbarrier pairs with phase bits; the k loop has no CTA barrier. The producer
// waits for stage q % 3 to be empty, splits k-block q into it, fences the generic-proxy stores to the async proxy and
// arrives on its full barrier. A consumer waits for the full barrier, loads and splits A, issues the wgmmas of q,
// wgmma.wait_group 1 (the wgmmas of q - 1 are done) and arrives on the empty barrier of q - 1's stage. The producer runs
// up to three k-blocks ahead, so while the consumers run a tile's epilogue it splits the next tile's first k-blocks.
// Shared-memory traffic per k-block in 3xTF32 (counted from the code): cp.async writes 24 KB (A 8, B 16), producer reads
// of raw B 16 KB, B hi/lo stores 32 KB, consumer reads of raw A 8 KB, wgmma B operand reads 96 KB (2 warpgroups x 2 k8 x
// 3 MMAs x 8 KB): 176 KB. With A split by the producer too it was 216 KB (A read back, A hi/lo stores 16 KB, A operand
// reads 24 KB), more than the 12 MMAs of the k-block take at the data-sheet tf32 rate.
// The epilogue works on the accumulator fragments in registers (bias / activation / activation-derivative mask /
// fused final linear layer, reduced over the four lanes that share a row) and stores 8-byte pairs; the four lanes of a
// row fill one 32-byte sector. The fused-head bias and weights are staged by the consumers behind a named barrier of
// their 256 threads.
// The k loop never writes the accumulators outside wgmma (they are zeroed before it and read after it), so ptxas adds no
// wgmma wait of its own and the loop's only wait is wait_group 1.
// ptxas (sm_90a): every variant runs its producer at 56 registers (FUSE 72) and its consumers at 224 (FUSE 216), no
// spills, no wgmma serialisation remark (C7513 / C7517). -Xptxas -v prints eight informational C7519 remarks per variant
// ("warpgroup.arrive is injected ... to allow use of registers in GMMA"), four per k-block of the two-way unrolled loop.
// Measured on an H100 80GB HBM3 (SXM, 700 W, 1980 MHz): 3xTF32 256 x 256 x 256 with G = 2048 takes 0.72-0.78 ms per
// layout (0.48 ms floor at data-sheet rates; 0.81-0.84 ms with A split by the producer through shared memory). See
// DESIGN.md §3.
#include "common.cuh"
#include <cstdio>
#include <cstdlib>

namespace {

constexpr int BM = 128, BN = 256, BK = 16;        // tile: 128 x 256 outputs; k-blocks of 16 floats (64-byte rows, SWIZZLE_64B)
constexpr int PRODUCER_THREADS = 128, CONSUMER_THREADS = 256;      // warpgroup 0 copies and splits, warpgroups 1 and 2 multiply
constexpr int THREADS = PRODUCER_THREADS + CONSUMER_THREADS;
// setmaxnreg: the launch gives every thread 65536 / 384 = 168 registers (rounded down to 8); the producer hands back all
// but 56 (72 with FUSE, whose first-layer evaluation spills below that) and the consumers take them: 128 x 56 + 256 x 224
// = 128 x 72 + 256 x 216 = 384 x 168. These are the smallest producer counts without spills (ptxas -v).
constexpr int LAUNCH_REGS = 168;
constexpr int producer_regs(bool fuse) { return fuse ? 72 : 56; }
constexpr int consumer_regs(bool fuse) { return (THREADS * LAUNCH_REGS - PRODUCER_THREADS * producer_regs(fuse)) / CONSUMER_THREADS; }
static_assert(THREADS * LAUNCH_REGS <= 65536 && consumer_regs(false) % 8 == 0 && consumer_regs(true) % 8 == 0, "tc_gemm: setmaxnreg split");
constexpr int CONSUMER_BAR = 1, PRODUCER_BAR = 2;                   // named barriers (0 is __syncthreads)
constexpr int A_BYTES = BM * BK * 4, B_BYTES = BN * BK * 4;          // 8 KB / 16 KB per k-block (raw A; B hi or lo copy)
constexpr int B_HI = 0, B_LO = B_BYTES;
constexpr int STAGE_BYTES = 2 * B_BYTES;                             // 32 KB hi/lo stage of B
constexpr int N_STAGES = 3;                                          // hi/lo stages: the producer splits up to two k-blocks ahead of the wgmmas in flight
constexpr int RAW_STAGES = 3;                                        // raw B ring: k-blocks in flight global -> shared memory
// A ring: raw fp32 A of a k-block, which the consumers load into wgmma register fragments and split there. The producer
// copies k-block q into slot q % A_STAGES (FUSE: computes it there) no earlier than its iteration q - RAW_STAGES, after
// waiting for the empty phase of k-block q - A_STAGES's stage; the consumers arrive on that phase only after loading
// the A fragments of k-block q - A_STAGES, the slot's previous content. So the stage barriers guard the A slots too, and
// the raw A is visible to the consumers through the full barrier of its k-block, like the hi/lo stage.
constexpr int A_STAGES = N_STAGES + RAW_STAGES;
// [rows, K] A: SWIZZLE_64B layout (A_BYTES). [K, rows] A: 16 k-rows of BM floats padded to A_T_LD, so that the k values
// t, t + 4 of a fragment load (t = lane % 4) fall 8 banks apart. FUSE computes [rows, K] A only.
constexpr int A_T_LD = BM + 8, A_T_BYTES = BK * A_T_LD * 4;
constexpr int a_slot_bytes(bool fuse) { return fuse ? A_BYTES : A_T_BYTES; }
constexpr int HEAD_MAX = 8;                                          // fused head: up to 8 output units (N = 1 critic, 2A <= 8 actor)
constexpr int HEAD_BYTES = (BN + HEAD_MAX * BN) * 4;                 // bias [256] + head weights [8][256]
// FUSE: the A operand is not loaded but COMPUTED — the previous (first) MLP layer relu(X W1^T + b1) with K0 <= 16 input
// columns, evaluated chunk by chunk straight into the swizzled operand tile — so the first hidden activation never
// round-trips HBM. W1 [256][16] (zero padded), b1 [256] and the tile's input rows [128][16] are staged once per tile.
constexpr int L1_MAXK = 16, L1_ROWS = 256;
constexpr int L1_W_BYTES = L1_ROWS * L1_MAXK * 4, L1_B_BYTES = L1_ROWS * 4, L1_X_BYTES = BM * L1_MAXK * 4;
constexpr int RAW_OFF = N_STAGES * STAGE_BYTES, A_OFF = RAW_OFF + RAW_STAGES * B_BYTES;
constexpr int head_off(bool fuse) { return A_OFF + A_STAGES * a_slot_bytes(fuse); }
constexpr int l1_off(bool fuse) { return head_off(fuse) + HEAD_BYTES; }
// The full / empty mbarrier pairs of the hi/lo stages sit in the BAR_BYTES just below the 512-byte aligned base (SWIZZLE_64B
// repeats every 512 bytes); with dynamic shared memory at least 16-byte aligned, barriers plus alignment take at most
// BAR_BYTES + 496 <= 1024 bytes.
constexpr int BAR_BYTES = 64;
static_assert(2 * N_STAGES * 8 <= BAR_BYTES && BAR_BYTES + 512 - 16 <= 1024, "tc_gemm: mbarrier area");
constexpr int smem_bytes(bool fuse) { return 1024 + l1_off(fuse) + (fuse ? L1_W_BYTES + L1_B_BYTES + L1_X_BYTES : 0); }  // the first-layer staging only where it is used
static_assert(smem_bytes(false) <= 227 * 1024 && smem_bytes(true) <= 227 * 1024, "tc_gemm: shared memory over the 227 KB per-CTA limit");

// ---- PTX wrappers ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const float* src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
// returns once the phase of parity `parity` has completed (the phase before the first counts as completed with parity 1)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n .reg .pred p;\n"
      "WAIT:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      " @!p bra WAIT;\n}" ::"r"(bar), "r"(parity) : "memory");
}
template <int ID, int N>
__device__ __forceinline__ void named_bar_sync() { asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(N) : "memory"); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// D (64 x 256, fp32, 128 registers per thread) += A (64 x 8, registers) * B (8 x 256, K-major in shared memory). The A
// fragment of warp w of the warpgroup, lane (g = lane / 4, t = lane % 4): a[0] = A[16 w + g][t], a[1] = A[16 w + g + 8][t],
// a[2] = A[16 w + g][t + 4], a[3] = A[16 w + g + 8][t + 4]. The registers must not change until the wgmma is complete.
__device__ __forceinline__ void wgmma_tf32(float (&d)[128], const uint32_t (&a)[4], uint64_t b_desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127 "
      "}, {%128, %129, %130, %131}, %132, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc));
}
// Shared-memory matrix descriptor of a K-major SWIZZLE_64B tile: start >> 4 | LBO >> 4 at bit 16 (unused by swizzled K-major
// layouts) | SBO >> 4 at bit 32 (512 B: the next 8-row atom) | layout type at bit 62 (2 = SWIZZLE_64B).
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(512 >> 4) << 32) | ((uint64_t)2 << 62);
}
// byte offset of 16-byte chunk `c` of row `r` inside a K-major SWIZZLE_64B tile (64-byte rows, 8-row atoms of 512 B;
// Swizzle<2,4,3>: chunk ^= (r / 2) % 4 — address bits [7,9) are (r >> 1) & 3)
__device__ __forceinline__ uint32_t sw64(int r, int c) { return (uint32_t)((r >> 3) * 512 + (r & 7) * 64 + ((c ^ ((r >> 1) & 3)) << 4)); }
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
// four 8 x 4 tiles of 32-bit words (8 x 8 of b16): lane l gives the address of row l % 8 of tile l / 8 and receives word
// l % 4 of row l / 4 of tile j in v[j]
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&v)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "r"(addr));
}
__device__ __forceinline__ uint32_t hi_of(uint32_t x) { return x & 0xFFFFE000u; }
__device__ __forceinline__ uint32_t lo_of(uint32_t x) { return __float_as_uint(__uint_as_float(x) - __uint_as_float(x & 0xFFFFE000u)); }
// hi_of and lo_of of a wgmma register operand, as one volatile asm: it stays where it is written, ahead of the
// wgmma.fence, instead of being sunk between the wgmmas (a definition of a wgmma input register inside the wgmma
// pipeline makes ptxas serialise the wgmmas)
__device__ __forceinline__ void split_reg(uint32_t x, uint32_t& hi, uint32_t& lo) {
  asm volatile("and.b32 %0, %2, 0xFFFFE000;\n\tsub.f32 %1, %2, %0;" : "=&r"(hi), "=r"(lo) : "r"(x));
}
// one 16-byte chunk (4 consecutive k of one row) into the hi tile and, for 3xTF32, the lo tile at the same offset
__device__ __forceinline__ void store_chunk(uint32_t hi_tile, uint32_t lo_tile, uint32_t off, uint4 v, bool split) {
  sts128(hi_tile + off, hi_of(v.x), hi_of(v.y), hi_of(v.z), hi_of(v.w));
  if (split) sts128(lo_tile + off, lo_of(v.x), lo_of(v.y), lo_of(v.z), lo_of(v.w));
}
// A 4 (k) x 4 (rows) block of an operand stored [K, rows]: v[k] holds rows 4 c4 .. 4 c4 + 3 at k = 4 kg + k. Transposed in
// registers into the four k-chunks of those rows. Row j of the block is stored at step (j - c4 / 2) % 4, so that the 8
// threads of a quarter warp (consecutive c4) write 8 rows with distinct r % 8, i.e. 8 distinct 16-byte bank groups.
__device__ __forceinline__ void store_block_t(uint32_t hi_tile, uint32_t lo_tile, int c4, int kg, const uint4 (&v)[4], bool split) {
  uint4 q0 = make_uint4(v[0].x, v[1].x, v[2].x, v[3].x), q1 = make_uint4(v[0].y, v[1].y, v[2].y, v[3].y);
  uint4 q2 = make_uint4(v[0].z, v[1].z, v[2].z, v[3].z), q3 = make_uint4(v[0].w, v[1].w, v[2].w, v[3].w);
  const int s = (c4 >> 1) & 3;
  if (s & 1) { const uint4 t = q0; q0 = q1; q1 = q2; q2 = q3; q3 = t; }
  if (s & 2) { uint4 t = q0; q0 = q2; q2 = t; t = q1; q1 = q3; q3 = t; }
  store_chunk(hi_tile, lo_tile, sw64(4 * c4 + (s & 3), kg), q0, split);
  store_chunk(hi_tile, lo_tile, sw64(4 * c4 + ((s + 1) & 3), kg), q1, split);
  store_chunk(hi_tile, lo_tile, sw64(4 * c4 + ((s + 2) & 3), kg), q2, split);
  store_chunk(hi_tile, lo_tile, sw64(4 * c4 + ((s + 3) & 3), kg), q3, split);
}

struct TcParams {
  GemmArgs g;
  int tiles_m;      // M / BM
  int split;        // 1: 3xTF32, 0: single TF32
  // EPI 4 (bias + ReLU + fused linear head): head_out[g, m, j] = sum_n head_w[g, j, n] * relu(C[g, m, n] + bias[n]) + head_b[g, j]
  const float* head_w;
  const float* head_b;
  float* head_out;
  int64_t head_gs, head_out_gs;  // group strides of head_w / head_b (same buffer family) and of head_out
  int head_n, store_c;           // head units (<= HEAD_MAX); store_c == 0: the hidden output itself is not needed (no backward)
  int head_js, head_ns;          // strides (floats) of head_w between head units j and between the BN contraction indices n: [head_n][BN] row-major = (BN, 1)
  TcFuseL1 l1;                   // FUSE: the first layer whose output is this product's A operand
};

// EPI: 0 plain store, 1 bias + relu, 2 relu-derivative mask, 3 generic (runtime bias / activation / mask), 5 relu-derivative mask from sign-bit words,
//      6 = 5 followed by a fused thin product of the masked tile (the input-gradient slice dX = dZ_0 W_1[:, cols], <= 8 columns; the tile itself is not stored),
//      4 bias + relu + fused linear head (the next, final layer of the MLP computed from the accumulator fragments in registers)
template <int EPI, bool FUSE = false>
__global__ void __launch_bounds__(THREADS, 1) tc_gemm_kernel(const TcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + BAR_BYTES + 511) & ~(uintptr_t)511);
  float* head_s = reinterpret_cast<float*>(smem + head_off(FUSE));  // [BN] bias then [HEAD_MAX][BN] head weights
  const uint32_t stage0 = smem_u32(smem), raw0 = stage0 + RAW_OFF, a0s = stage0 + A_OFF;
  const uint32_t full0 = stage0 - BAR_BYTES, empty0 = full0 + N_STAGES * 8;  // mbarriers of hi/lo stage s: full0 + 8 s, empty0 + 8 s
  const uint32_t w1s = stage0 + l1_off(FUSE), b1s = w1s + L1_W_BYTES, xs = b1s + L1_B_BYTES;
  auto a_slot = [&](int q) { return a0s + (uint32_t)(q % A_STAGES) * (uint32_t)a_slot_bytes(FUSE); };
  const bool a_km = FUSE || p.g.a_kmajor != 0;  // A stored [rows, K] (else [K, rows])

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const GemmArgs& g = p.g;
  const int nkb = g.K / BK, tiles_m = p.tiles_m;
  const int my_tiles = (g.G * tiles_m - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;  // tiles blockIdx.x + i gridDim.x
  const int nq = my_tiles * nkb;                                                                // this CTA's k-block stream
  auto tile_of = [&](int i) { return (int)blockIdx.x + i * (int)gridDim.x; };

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < N_STAGES; ++s) {
      mbar_init(full0 + 8 * s, PRODUCER_THREADS);
      mbar_init(empty0 + 8 * s, CONSUMER_THREADS);
    }
  }
  __syncthreads();  // the only CTA-wide barrier: the mbarriers are initialised

  if (wg == 0) {
    // ================= producer warpgroup: copy and split the k-block stream =================
    setmaxnreg_dec<producer_regs(FUSE)>();
    const bool b_km = g.b_kmajor != 0, split = p.split != 0;
    // Per-thread chunks of one k-block, in a map of 256 slots: producer thread pt works slots v = pt and v = pt + 128.
    // stored [rows, K]: 16-byte chunk fc of rows fr + 64 j (A: j < 2, B: j < 4), fr = v / 4, fc = v % 4
    // stored [K, rows]: B: 4 x 4 blocks, rows 4 c4 .. 4 c4 + 3 at k = 4 kg .. 4 kg + 3; A: in slots v < 128, the chunks
    //                   of rows 4 c4 .. 4 c4 + 3 at k = 4 kg .. 4 kg + 3 (c4 = v % 32, kg = v / 32)
    // B: slot v's chunk j sits at (256 j + v) * 16 of the raw B slot, so the copies and the reads back of a warp are 512
    // contiguous bytes. A thread reads back exactly the B chunks it copied, so cp.async.wait_group is all the visibility
    // the raw B ring needs (no mbarrier, no barrier of the warpgroup). A: copied straight into the consumers' layout
    // (SWIZZLE_64B, or k-rows of A_T_LD floats) and never read back by the producer.
    constexpr int MAP = 2 * PRODUCER_THREADS;
    const int pt = tid;

    auto copy_kb = [&](int q) {  // k-block q of the stream: raw chunks global -> raw B slot q % RAW_STAGES and A slot q % A_STAGES; always one commit group
      if (q < nq) {
        const int t = tile_of(q / nkb), kb = q % nkb, grp = t / tiles_m, m0 = (t % tiles_m) * BM;
        const float* A = g.A + (int64_t)(grp / g.a_gdiv) * g.a_gs;
        const float* Bg = g.B + (int64_t)(grp / g.b_gdiv) * g.b_gs;
        const uint32_t as = a_slot(q);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int v = pt + h * PRODUCER_THREADS, fr = v >> 2, fc = v & 3;
          const uint32_t raw = raw0 + (uint32_t)(q % RAW_STAGES) * B_BYTES + (uint32_t)v * 16u;
          if (!FUSE) {
            if (a_km) {
              const float* src = A + (int64_t)(m0 + fr) * g.lda + kb * BK + fc * 4;
              cp_async16(as + sw64(fr, fc), src);
              cp_async16(as + sw64(fr, fc) + 4096u, src + (int64_t)64 * g.lda);  // rows fr + 64: 8 atoms further
            } else if (h == 0) {
              const int c4 = v & 31, kg = v >> 5;
              const float* src = A + (int64_t)(kb * BK + kg * 4) * g.lda + m0 + c4 * 4;
#pragma unroll
              for (int k = 0; k < 4; ++k) cp_async16(as + (uint32_t)(((kg * 4 + k) * A_T_LD + c4 * 4) * 4), src + (int64_t)k * g.lda);
            }
          }
          const float* src = b_km ? Bg + (int64_t)fr * g.ldb + kb * BK + fc * 4 : Bg + (int64_t)(kb * BK + (v >> 6) * 4) * g.ldb + (v & 63) * 4;
          const int64_t step = b_km ? (int64_t)64 * g.ldb : (int64_t)g.ldb;  // next chunk j: 64 rows further / the next k
#pragma unroll
          for (int j = 0; j < 4; ++j) cp_async16(raw + j * MAP * 16, src + j * step);
        }
      }
      cp_async_commit();
    };

    auto split_kb = [&](int q, int s) {  // k-block q: split the raw B chunks this thread copied into hi/lo stage s (FUSE: and compute the A chunks into A slot q)
      const uint32_t st = stage0 + (uint32_t)s * STAGE_BYTES;
#pragma unroll(FUSE ? 1 : 2)  // the first-layer evaluation of both slots at once would not fit the producer's registers
      for (int h = 0; h < 2; ++h) {
        const int v = pt + h * PRODUCER_THREADS, fr = v >> 2, fc = v & 3;
        const uint32_t raw = raw0 + (uint32_t)(q % RAW_STAGES) * B_BYTES + (uint32_t)v * 16u;
        const uint32_t km_off = sw64(fr, fc);  // rows fr + 64 j: + j * 4096 bytes (64 rows = 8 atoms)
        if (FUSE) {
          // A chunk values: relu(b1[k] + sum_j x[j] W1[k][j]) for k = 16 kb + 4 fc + {0..3}, rows fr and fr + 64
          const int kb = q % nkb, k0 = kb * BK + fc * 4;
          const uint4 bq = lds128(b1s + (uint32_t)k0 * 4u);
          float c0[4] = {__uint_as_float(bq.x), __uint_as_float(bq.y), __uint_as_float(bq.z), __uint_as_float(bq.w)};
          float c1[4] = {c0[0], c0[1], c0[2], c0[3]};
          const int np = (p.l1.x_k + 3) >> 2;
#pragma unroll
          for (int c4 = 0; c4 < L1_MAXK / 4; ++c4) {
            if (c4 < np) {
              const uint4 x0 = lds128(xs + sw64(fr, c4)), x1 = lds128(xs + sw64(fr + 64, c4));
#pragma unroll
              for (int qq = 0; qq < 4; ++qq) {
                const uint4 w = lds128(w1s + (uint32_t)((k0 + qq) * 64 + ((c4 ^ fc) << 4)));  // W1 row k: chunk c4 at c4 ^ ((k >> 2) & 3)
                c0[qq] = fmaf(__uint_as_float(x0.x), __uint_as_float(w.x), c0[qq]); c1[qq] = fmaf(__uint_as_float(x1.x), __uint_as_float(w.x), c1[qq]);
                c0[qq] = fmaf(__uint_as_float(x0.y), __uint_as_float(w.y), c0[qq]); c1[qq] = fmaf(__uint_as_float(x1.y), __uint_as_float(w.y), c1[qq]);
                c0[qq] = fmaf(__uint_as_float(x0.z), __uint_as_float(w.z), c0[qq]); c1[qq] = fmaf(__uint_as_float(x1.z), __uint_as_float(w.z), c1[qq]);
                c0[qq] = fmaf(__uint_as_float(x0.w), __uint_as_float(w.w), c0[qq]); c1[qq] = fmaf(__uint_as_float(x1.w), __uint_as_float(w.w), c1[qq]);
              }
            }
          }
          const uint4 a0 = make_uint4(__float_as_uint(fmaxf(c0[0], 0.f)), __float_as_uint(fmaxf(c0[1], 0.f)), __float_as_uint(fmaxf(c0[2], 0.f)), __float_as_uint(fmaxf(c0[3], 0.f)));
          const uint4 a1 = make_uint4(__float_as_uint(fmaxf(c1[0], 0.f)), __float_as_uint(fmaxf(c1[1], 0.f)), __float_as_uint(fmaxf(c1[2], 0.f)), __float_as_uint(fmaxf(c1[3], 0.f)));
          const uint32_t as = a_slot(q);  // raw, like a copied A: the consumers split it
          sts128(as + km_off, a0.x, a0.y, a0.z, a0.w);
          sts128(as + km_off + 4096u, a1.x, a1.y, a1.z, a1.w);
          if (p.l1.store) {  // the first hidden activation, for the backward pass
            const int t = tile_of(q / nkb);
            float* hs = p.l1.store + (int64_t)(t / tiles_m) * p.l1.store_gs + (int64_t)((t % tiles_m) * BM + fr) * g.K + k0;
            *reinterpret_cast<uint4*>(hs) = a0;
            *reinterpret_cast<uint4*>(hs + (int64_t)64 * g.K) = a1;
          }
        }
        if (b_km) {
#pragma unroll
          for (int j = 0; j < 4; ++j) store_chunk(st + B_HI, st + B_LO, km_off + (uint32_t)j * 4096u, lds128(raw + j * MAP * 16), split);
        } else {
          uint4 vb[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) vb[k] = lds128(raw + k * MAP * 16);
          store_block_t(st + B_HI, st + B_LO, v & 63, v >> 6, vb, split);
        }
      }
    };

    auto stage_l1 = [&](int t) {  // FUSE: first-layer parameters and input rows of tile t
      const int grp = t / tiles_m, m0 = (t % tiles_m) * BM, xk = p.l1.x_k;
      const float* w1 = p.l1.w1 + (int64_t)grp * p.l1.gs;
      const float* b1 = p.l1.b1 + (int64_t)grp * p.l1.gs;
      const float* x = p.l1.x + (int64_t)(grp / p.l1.x_gdiv) * p.l1.x_gs + (int64_t)m0 * p.l1.x_ld;
      float* w1f = reinterpret_cast<float*>(smem + l1_off(FUSE));
      float* b1f = reinterpret_cast<float*>(smem + l1_off(FUSE) + L1_W_BYTES);
      float* xf = reinterpret_cast<float*>(smem + l1_off(FUSE) + L1_W_BYTES + L1_B_BYTES);
#pragma unroll 1  // rolled: once per tile, and the producer has few registers
      for (int i = pt; i < L1_ROWS * L1_MAXK; i += PRODUCER_THREADS) {  // zero-padded to [256][16]
        const int k = i / L1_MAXK, j = i % L1_MAXK;
        w1f[k * L1_MAXK + ((((j >> 2) ^ ((k >> 2) & 3)) << 2) | (j & 3))] = (k < g.K && j < xk) ? __ldg(w1 + (int64_t)k * xk + j) : 0.f;
      }
      for (int i = pt; i < L1_ROWS; i += PRODUCER_THREADS) b1f[i] = i < g.K ? __ldg(b1 + i) : 0.f;
#pragma unroll 1
      for (int i = pt; i < BM * L1_MAXK; i += PRODUCER_THREADS) {
        const int r = i / L1_MAXK, j = i % L1_MAXK;
        xf[(sw64(r, j >> 2) >> 2) + (j & 3)] = j < xk ? __ldg(x + (int64_t)r * p.l1.x_ld + j) : 0.f;
      }
    };

    // Per k-block q: wait until stage s is empty (the consumers' wgmmas of q - N_STAGES are done), wait for this thread's
    // chunks of q, split them into stage s, mark it full and copy q + RAW_STAGES into the raw slot just read back. The
    // producer runs up to N_STAGES k-blocks ahead of the wgmmas, across tile boundaries, so the next tile's first stages
    // are split while the consumers run this tile's epilogue.
#pragma unroll 1
    for (int q = 0; q < RAW_STAGES; ++q) copy_kb(q);
    int s = 0;
    uint32_t ph = 1;  // parity of the empty phase to wait for: the first pass over the stages finds them empty
#pragma unroll 1
    for (int q = 0; q < nq; ++q) {
      if (FUSE && q % nkb == 0) {  // the first k-block of a tile: its first-layer staging, once every split of the previous tile is done
        if (q > 0) named_bar_sync<PRODUCER_BAR, PRODUCER_THREADS>();
        stage_l1(tile_of(q / nkb));
        named_bar_sync<PRODUCER_BAR, PRODUCER_THREADS>();
      }
      mbar_wait(empty0 + 8 * s, ph);
      cp_async_wait<RAW_STAGES - 1>();  // this thread's chunks of k-block q
      split_kb(q, s);
      fence_proxy_async();              // the generic-proxy stores -> visible to the tensor core (async proxy)
      mbar_arrive(full0 + 8 * s);
      copy_kb(q + RAW_STAGES);
      if (++s == N_STAGES) { s = 0; ph ^= 1; }
    }
    cp_async_wait<0>();  // the trailing (empty) commit groups
    return;
  }

  // ================= consumer warpgroups 1 and 2: wgmma and the epilogue =================
  // Consumer warpgroup cw owns rows [64 cw, 64 cw + 64) of the tile. Per k-block: wait until its stage is full, load the
  // raw A fragments of its rows from the A slot and split them in registers, issue the wgmmas (A from registers, B from
  // the hi/lo stage), wgmma.wait_group 1 (the wgmmas of the previous k-block are done) and release that previous stage.
  // A register operand must not change while its wgmma is in flight, so consecutive k-blocks use the two fragment sets
  // af[0] and af[1] in turn (the k loop is unrolled by two). In the SASS ptxas folds most of the second set onto the
  // first: the runtime `split` branch ends each k-block in four gsb0-terminated HGMMA chains, and wait_group 1 leaves
  // only the last (hi x hi of the second k8) in flight, so only its hi registers get a separate copy. It also means
  // only about one of a k-block's six MMAs overlaps the issue of the next k-block.
  // The k loop never writes the accumulators outside wgmma (they are zeroed before it and read after it), so nothing in
  // it makes ptxas wait for the wgmmas in flight.
  setmaxnreg_inc<consumer_regs(FUSE)>();
  const int cw = wg - 1, ct = tid - PRODUCER_THREADS;
  const uint64_t b_desc0 = make_desc(stage0);
  const bool split = p.split != 0;
  // Per-thread offsets of the A fragment inside an A slot (rows of this warp: 64 cw + 16 (warp % 4) + {g, g + 8}).
  // [rows, K]: two ldmatrix.x4 per k-block, one per k8 kk; tile j = lane / 8 is rows + 8 (j % 2) at chunk 2 kk + j / 2, so
  // v[j] is the fragment's a[j]. The 8 rows of a tile sit in 8 distinct 16-byte bank groups (SWIZZLE_64B).
  // [K, rows]: a[j] of k8 kk is row g + 8 (j % 2) at k = 8 kk + 4 (j / 2) + t, 4 bytes each; the k-row pitch of A_T_LD
  // floats puts the four t of a row 8 banks apart.
  const int wrow = cw * 64 + (warp & 3) * 16, g8 = lane >> 2, t4 = lane & 3;
  const uint32_t lm_off = sw64(wrow + (lane & 7) + 8 * ((lane >> 3) & 1), lane >> 4);  // ^ 32: chunk + 2 (chunks 0 and 1 here; the swizzle XORs bits 4-5 only)
  const uint32_t t_off = (uint32_t)((t4 * A_T_LD + wrow + g8) * 4);
  uint32_t af[2][2][BK / 8][4];  // [fragment set][hi, lo][k8][a0..a3]
  float acc[128];
  auto kblock = [&](int q, int s, uint32_t (&f)[2][BK / 8][4]) {
    const uint32_t as = a_slot(q), cur = (uint32_t)s * STAGE_BYTES;
#pragma unroll
    for (int kk = 0; kk < BK / 8; ++kk) {
      uint32_t x[4];
      if (a_km) {
        ldsm_x4(as + (lm_off ^ (uint32_t)(kk * 32)), x);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) x[j] = lds32(as + t_off + (uint32_t)(((8 * kk + 4 * (j >> 1)) * A_T_LD + 8 * (j & 1)) * 4));
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) split_reg(x[j], f[0][kk][j], f[1][kk][j]);
    }
    wgmma_fence();  // the fragment registers are written before the wgmmas read them
#pragma unroll
    for (int kk = 0; kk < BK / 8; ++kk) {  // per MMA (K = 8 tf32): 32 bytes further inside the swizzled 64-byte rows
      const uint32_t o = cur + kk * 32;
      const uint64_t bh = b_desc0 + ((o + B_HI) >> 4), bl = b_desc0 + ((o + B_LO) >> 4);
      if (split) {
        wgmma_tf32(acc, f[1][kk], bh);
        wgmma_tf32(acc, f[0][kk], bl);
      }
      wgmma_tf32(acc, f[0][kk], bh);
    }
    wgmma_commit();
  };
  int s = 0, q = 0;  // q: this CTA's k-block stream
  uint32_t ph = 0;   // parity of the full phase to wait for
#pragma unroll 1
  for (int i = 0; i < my_tiles; ++i) {
#pragma unroll
    for (int j = 0; j < 128; ++j) acc[j] = 0.f;
    int prev = 0;
    auto step = [&](int kb, uint32_t (&f)[2][BK / 8][4]) {
      mbar_wait(full0 + 8 * s, ph);
      kblock(q, s, f);
      wgmma_wait<1>();                               // the wgmmas of the previous k-block are done
      if (kb > 0) mbar_arrive(empty0 + 8 * prev);   // ... so its stage is free for the producer
      prev = s;
      ++q;
      if (++s == N_STAGES) { s = 0; ph ^= 1; }
    };
#pragma unroll 1
    for (int kb = 0; kb < nkb; kb += 2) {
      step(kb, af[0]);
      if (kb + 1 < nkb) step(kb + 1, af[1]);
    }

    // ---- epilogue of tile i: acc[4 c + {0, 1}] = row r0, columns 8 c + 2 (lane % 4) + {0, 1}; acc[4 c + {2, 3}] = row r0 + 8 ----
    const int t = tile_of(i), grp = t / tiles_m, m0 = (t % tiles_m) * BM;
    if (EPI == 4 || EPI == 6) {  // this tile's fused-head bias / weights, staged while the last wgmmas finish, once both consumer
                                 // warpgroups are done reading the previous tile's; BN == CONSUMER_THREADS: element ct of each row
      named_bar_sync<CONSUMER_BAR, CONSUMER_THREADS>();
      const float* wsrc = p.head_w + (int64_t)grp * p.head_gs;
      if (EPI == 4) head_s[ct] = __ldg(g.bias + (int64_t)grp * g.bias_gs + ct);
#pragma unroll
      for (int j = 0; j < HEAD_MAX; ++j)
        if (j < p.head_n) head_s[BN + j * BN + ct] = __ldg(wsrc + (int64_t)j * p.head_js + (int64_t)ct * p.head_ns);
    }
    wgmma_wait<0>();
    mbar_arrive(empty0 + 8 * prev);
    if (EPI == 4 || EPI == 6) named_bar_sync<CONSUMER_BAR, CONSUMER_THREADS>();
    const int r0 = m0 + cw * 64 + (warp & 3) * 16 + (lane >> 2), cl = (lane & 3) * 2;
    float* C = g.C + (int64_t)grp * g.c_gs + (int64_t)r0 * g.ldc + cl;
    const int64_t c8 = (int64_t)8 * g.ldc;
    const float* bias = (EPI == 1 || (EPI == 3 && g.bias)) ? g.bias + (int64_t)grp * g.bias_gs + cl : nullptr;
    const float* mask = (EPI == 2 || (EPI == 3 && g.mask)) ? g.mask + (int64_t)grp * g.mask_gs + (int64_t)r0 * g.ldmask + cl : nullptr;
    const int64_t m8 = (int64_t)8 * g.ldmask;
    const uint32_t* mbits = (EPI == 5 || EPI == 6) ? g.mask_bits + (int64_t)grp * g.mask_bits_gs + (int64_t)r0 * (BN / 32) : nullptr;
    uint32_t word0 = 0, word1 = 0;  // sign-bit words of the two rows: read (EPI 5 / 6) or built (EPI 4) 32 columns at a time
#pragma unroll
    for (int c = 0; c < BN / 8; ++c) {
      float v00 = acc[4 * c], v01 = acc[4 * c + 1], v10 = acc[4 * c + 2], v11 = acc[4 * c + 3];
      const int col = 8 * c, bit = (c & 3) * 8 + cl;  // column of v*0 is col + cl; its bit inside the 32-column word
      if (EPI == 5 || EPI == 6) {  // ReLU derivative from the sign-bit words the forward kernel wrote
        if ((c & 3) == 0) { word0 = __ldg(mbits + (c >> 2)); word1 = __ldg(mbits + 8 * (BN / 32) + (c >> 2)); }
        v00 = (word0 >> bit) & 1u ? v00 : 0.f; v01 = (word0 >> (bit + 1)) & 1u ? v01 : 0.f;
        v10 = (word1 >> bit) & 1u ? v10 : 0.f; v11 = (word1 >> (bit + 1)) & 1u ? v11 : 0.f;
      }
      if (EPI == 4) {
        const float2 b = *reinterpret_cast<const float2*>(head_s + col + cl);
        v00 = fmaxf(v00 + b.x, 0.f); v01 = fmaxf(v01 + b.y, 0.f); v10 = fmaxf(v10 + b.x, 0.f); v11 = fmaxf(v11 + b.y, 0.f);
        if (g.bits_out) {  // sign bits of the hidden outputs: all a dX-only backward pass needs of them (1/32 of the bytes)
          if ((c & 3) == 0) word0 = word1 = 0;
          word0 |= (v00 > 0.f ? 1u : 0u) << bit | (v01 > 0.f ? 1u : 0u) << (bit + 1);
          word1 |= (v10 > 0.f ? 1u : 0u) << bit | (v11 > 0.f ? 1u : 0u) << (bit + 1);
          if ((c & 3) == 3) {  // the four lanes of a row hold 8 bits each of the word
            word0 |= __shfl_xor_sync(0xffffffffu, word0, 1); word0 |= __shfl_xor_sync(0xffffffffu, word0, 2);
            word1 |= __shfl_xor_sync(0xffffffffu, word1, 1); word1 |= __shfl_xor_sync(0xffffffffu, word1, 2);
            if ((lane & 3) == 0) {
              uint32_t* bo = g.bits_out + (int64_t)grp * g.bits_out_gs + (int64_t)r0 * (BN / 32) + (c >> 2);
              bo[0] = word0;
              bo[8 * (BN / 32)] = word1;
            }
          }
        }
      }
      if (EPI == 4 || EPI == 6) {  // the fragment the thin product below reads, in place
        acc[4 * c] = v00; acc[4 * c + 1] = v01; acc[4 * c + 2] = v10; acc[4 * c + 3] = v11;
        if (!p.store_c) continue;
      }
      if (EPI == 1) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(bias + col));
        v00 = fmaxf(v00 + b.x, 0.f); v01 = fmaxf(v01 + b.y, 0.f); v10 = fmaxf(v10 + b.x, 0.f); v11 = fmaxf(v11 + b.y, 0.f);
      } else if (EPI == 2) {
        const float2 ma = __ldg(reinterpret_cast<const float2*>(mask + col)), mb = __ldg(reinterpret_cast<const float2*>(mask + m8 + col));
        v00 = ma.x > 0.f ? v00 : 0.f; v01 = ma.y > 0.f ? v01 : 0.f; v10 = mb.x > 0.f ? v10 : 0.f; v11 = mb.y > 0.f ? v11 : 0.f;
      } else if (EPI == 3) {
        if (bias) {
          const float2 b = __ldg(reinterpret_cast<const float2*>(bias + col));
          v00 += b.x; v01 += b.y; v10 += b.x; v11 += b.y;
        }
        if (g.act >= 0) { v00 = act_apply(v00, g.act); v01 = act_apply(v01, g.act); v10 = act_apply(v10, g.act); v11 = act_apply(v11, g.act); }
        if (mask) {
          const float2 ma = __ldg(reinterpret_cast<const float2*>(mask + col)), mb = __ldg(reinterpret_cast<const float2*>(mask + m8 + col));
          v00 *= act_grad_from_output(ma.x, g.mask_act); v01 *= act_grad_from_output(ma.y, g.mask_act);
          v10 *= act_grad_from_output(mb.x, g.mask_act); v11 *= act_grad_from_output(mb.y, g.mask_act);
        }
      }
      *reinterpret_cast<float2*>(C + col) = make_float2(v00, v01);
      *reinterpret_cast<float2*>(C + c8 + col) = make_float2(v10, v11);
    }
    if (EPI == 4 || EPI == 6) {  // the next (thin) product on the fragment, one head unit at a time: h[j] = sum_c v[c] * W[j][c]
      float* ho = p.head_out + (int64_t)grp * p.head_out_gs + (int64_t)r0 * p.head_n;
      const float* hb = p.head_b ? p.head_b + (int64_t)grp * p.head_gs : nullptr;
#pragma unroll 1
      for (int j = 0; j < HEAD_MAX; ++j) {
        if (j < p.head_n) {
          float s0 = 0.f, s1 = 0.f;  // the four lanes of a row each sum a quarter of the columns, in column order
#pragma unroll
          for (int c = 0; c < BN / 8; ++c) {
            const float2 w = *reinterpret_cast<const float2*>(head_s + BN + j * BN + 8 * c + cl);
            s0 = fmaf(acc[4 * c], w.x, s0); s0 = fmaf(acc[4 * c + 1], w.y, s0);
            s1 = fmaf(acc[4 * c + 2], w.x, s1); s1 = fmaf(acc[4 * c + 3], w.y, s1);
          }
          s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
          s1 += __shfl_xor_sync(0xffffffffu, s1, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
          if ((lane & 3) == 0) {
            const float b = hb ? __ldg(hb + j) : 0.f;
            ho[j] = s0 + b;
            ho[(int64_t)8 * p.head_n + j] = s1 + b;
          }
        }
      }
    }
  }
}


// bias gradient for the dW products routed to the tensor-core engine: out[g, n] = sum_b dY[g, b, n]
__global__ void colsum_kernel(const float* __restrict__ A, int64_t a_gs, int a_gdiv, int lda, int K, int M, float* __restrict__ out, int64_t out_gs) {
  const int g = blockIdx.y, m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float* a = A + (int64_t)(g / a_gdiv) * a_gs + m;
  float s = 0.f;
  for (int k = 0; k < K; ++k) s += a[(int64_t)k * lda];
  out[(int64_t)g * out_gs + m] = s;
}

}  // namespace

bool tc_gemm_eligible(const GemmArgs& a) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (a.M % BM != 0 || a.N != BN || a.K % BK != 0 || a.accumulate) return false;
  if (a.a_kmajor == 0 && a.b_kmajor != 0) return false;
  if (!al16(a.A) || !al16(a.B) || !al16(a.C) || a.lda % 4 || a.ldb % 4 || a.ldc % 4 || a.a_gs % 4 || a.b_gs % 4 || a.c_gs % 4) return false;
  if (a.bias && (!al16(a.bias) || a.bias_gs % 4)) return false;
  if (a.mask && (!al16(a.mask) || a.ldmask % 4 || a.mask_gs % 4)) return false;
  return true;
}

template <int EPI, bool FUSE = false>
int tc_set_attr() {
  IL_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<EPI, FUSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(FUSE)));
  return 0;
}

int tc_gemm_init() {
  IL_TRY((tc_set_attr<0>())); IL_TRY((tc_set_attr<1>())); IL_TRY((tc_set_attr<2>())); IL_TRY((tc_set_attr<3>())); IL_TRY((tc_set_attr<4>()));
  IL_TRY((tc_set_attr<4, true>())); IL_TRY((tc_set_attr<5>())); IL_TRY((tc_set_attr<6>()));
  return 0;
}

// persistent: one CTA per SM, striding over the 128 x 256 tiles. The tiles of a group are adjacent and a wave holds whole
// groups (the grid is a multiple of tiles_m), so a group's B operand is read from HBM once and from L2 after that.
template <int EPI, bool FUSE = false>
static int tc_launch(il_handle* h, TcParams& p, cudaStream_t stream) {
  const GemmArgs& a = p.g;
  p.tiles_m = a.M / BM;
  const int tiles = a.G * p.tiles_m, wave = h->sm_count >= p.tiles_m ? h->sm_count / p.tiles_m * p.tiles_m : h->sm_count;
  IL_LAUNCH(h, (tc_gemm_kernel<EPI, FUSE>), tiles < wave ? tiles : wave, THREADS, smem_bytes(FUSE), stream, p);
  return 0;
}

bool tc_head_fusable(const il_handle* h, const GemmArgs& a, int head_n) {
  return h->gemm_mode != IL_GEMM_FP32 && tc_gemm_eligible(a) && a.bias && a.act == IL_ACT_RELU && !a.mask && !a.colsum && head_n >= 1 && head_n <= HEAD_MAX;
}

// The first layer can be computed in place of the A operand loads when the staging buffers fit: K0 <= 16 input columns and
// hidden width (the K of the dense product) <= 256.
bool tc_l1_fusable(const il_handle* h, const GemmArgs& a, int x_k) {
  return h->tc_fuse_l1 && tc_gemm_eligible(a) && x_k >= 1 && x_k <= L1_MAXK && a.K <= L1_ROWS && a.a_kmajor;
}

int launch_tc_gemm_head(il_handle* h, const GemmArgs& a, const float* head_w, const float* head_b, int64_t head_gs, int head_n, float* head_out, int64_t head_out_gs, int store_c,
                        cudaStream_t stream, const TcFuseL1* l1) {
  IL_CHECK(tc_head_fusable(h, a, head_n), "tc_gemm_head: not fusable");
  TcParams p{};
  p.g = a;
  p.split = h->gemm_mode == IL_GEMM_TF32X3 ? 1 : 0;
  p.head_w = head_w; p.head_b = head_b; p.head_out = head_out; p.head_gs = head_gs; p.head_out_gs = head_out_gs; p.head_n = head_n; p.store_c = store_c;
  p.head_js = BN; p.head_ns = 1;
  double bytes = gemm_algorithmic_bytes(a, store_c != 0) + 4.0 * a.G * (double)a.M * head_n, flops = 2.0 * a.M * a.N * a.K * a.G;
  if (l1) {
    IL_CHECK(tc_l1_fusable(h, a, l1->x_k), "tc_gemm_head: first layer not fusable (K0=%d)", l1->x_k);
    IL_CHECK(l1->x && l1->w1 && l1->b1 && (reinterpret_cast<uintptr_t>(l1->b1) & 15) == 0 && l1->gs % 4 == 0, "tc_gemm_head: bad first-layer buffers");
    IL_CHECK(!l1->store || ((reinterpret_cast<uintptr_t>(l1->store) & 15) == 0 && l1->store_gs % 4 == 0), "tc_gemm_head: unaligned hidden store");
    p.l1 = *l1;
    // algorithmic traffic: the A operand is not read; X, W1, b1 are, and the hidden store (if any) is written
    const double gx = (a.G + l1->x_gdiv - 1) / l1->x_gdiv;
    bytes += -4.0 * a.G * (double)a.M * a.K + 4.0 * (gx * a.M * l1->x_k + (double)a.G * a.K * (l1->x_k + 1)) + (l1->store ? 4.0 * a.G * (double)a.M * a.K : 0.0);
    flops += 2.0 * a.G * (double)a.M * a.K * l1->x_k;
  }
  auto run = [&]() { return l1 ? tc_launch<4, true>(h, p, stream) : tc_launch<4>(h, p, stream); };
  if (h->profiling) {  // the fused layer-2 + head launches are dense-layer launches too (head flops / bytes are negligible)
    ProfiledLaunch pl;
    IL_TRY(profile_open(h, &pl, flops, bytes, stream));
    const int rc = run();
    IL_TRY(profile_close(h, &pl, stream));
    return rc;
  }
  return run();
}

// dX-only backward of a depth-2 ReLU net in one launch: T = (A B) * relu'(bits) on the tensor cores (never stored), then out[g, m, j] = sum_n T[m, n] w[n * w_ns + j]
// for head_n <= 8 columns in the epilogue (the input-gradient slice of the first layer, training.py:36-41).
bool tc_dx_head_fusable(const il_handle* h, const GemmArgs& a, int head_n) {
  return h->gemm_mode != IL_GEMM_FP32 && a.M >= 128 && a.K >= 128 && tc_gemm_eligible(a) && a.mask_bits && !a.mask && !a.bias && a.act < 0 && !a.colsum && a.mask_act == IL_ACT_RELU &&
         head_n >= 1 && head_n <= HEAD_MAX;
}
int launch_tc_gemm_dx_head(il_handle* h, const GemmArgs& a, const float* w, int64_t w_gs, int w_ns, int head_n, float* out, int64_t out_gs, cudaStream_t stream) {
  IL_CHECK(tc_dx_head_fusable(h, a, head_n), "tc_gemm_dx_head: not fusable");
  TcParams p{};
  p.g = a;
  p.split = h->gemm_mode == IL_GEMM_TF32X3 ? 1 : 0;
  p.head_w = w; p.head_b = nullptr; p.head_out = out; p.head_gs = w_gs; p.head_out_gs = out_gs; p.head_n = head_n; p.store_c = 0;
  p.head_js = 1; p.head_ns = w_ns;
  const double bytes = gemm_algorithmic_bytes(a, false) + 4.0 * a.G * (double)a.M * head_n, flops = 2.0 * a.M * a.N * a.K * a.G;
  if (h->profiling) {
    ProfiledLaunch pl;
    IL_TRY(profile_open(h, &pl, flops, bytes, stream));
    const int rc = tc_launch<6>(h, p, stream);
    IL_TRY(profile_close(h, &pl, stream));
    return rc;
  }
  return tc_launch<6>(h, p, stream);
}

int launch_tc_gemm(il_handle* h, const GemmArgs& a, cudaStream_t stream) {
  IL_CHECK(tc_gemm_eligible(a), "tc_gemm: shape/layout not eligible (M=%d N=%d K=%d)", a.M, a.N, a.K);
  TcParams p{};
  p.g = a;
  p.split = h->gemm_mode == IL_GEMM_TF32X3 ? 1 : 0;
  const bool bits = a.mask_bits != nullptr;  // sign-bit mask: takes precedence over an fp32 mask of the same activation
  IL_CHECK(!bits || (!a.bias && a.act < 0 && a.mask_act == IL_ACT_RELU), "tc_gemm: sign-bit masks are the ReLU derivative of a plain product");
  if (bits) p.g.mask = nullptr;
  const bool plain = !a.bias && a.act < 0 && !a.mask && !bits;
  const bool bias_relu = a.bias && a.act == IL_ACT_RELU && !a.mask;
  const bool mask_relu = !a.bias && a.act < 0 && a.mask && a.mask_act == IL_ACT_RELU && !bits;
  if (bits) IL_TRY(tc_launch<5>(h, p, stream));
  else if (plain) IL_TRY(tc_launch<0>(h, p, stream));
  else if (bias_relu) IL_TRY(tc_launch<1>(h, p, stream));
  else if (mask_relu) IL_TRY(tc_launch<2>(h, p, stream));
  else IL_TRY(tc_launch<3>(h, p, stream));
  if (a.colsum) {
    dim3 cg((a.M + 127) / 128, a.G);
    IL_LAUNCH(h, colsum_kernel, cg, 128, 0, stream, a.A, a.a_gs, a.a_gdiv, a.lda, a.K, a.M, a.colsum, a.colsum_gs);
  }
  return 0;
}
