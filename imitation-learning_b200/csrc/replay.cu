// ReplayMemory (memory.py:12-68) as packed 16-byte-aligned rows per replica: append / absorbing wrap, index
// sampling, gather, and the mixed-batch overwrite (models.py:287-290).
#include "common.cuh"

namespace {

__device__ __forceinline__ void write_row(float* dst, const RowLayout& L, int S, int A, int lane, const float* state, const float* action, float reward, const float* next_state,
                                          float terminal, float timeout, float step, bool state_absorbing, bool next_absorbing) {
  for (int j = lane; j < S; j += 32) {
    dst[L.state + j] = state_absorbing ? (j == S - 1 ? 1.f : 0.f) : state[j];
    dst[L.next_state + j] = next_absorbing ? (j == S - 1 ? 1.f : 0.f) : next_state[j];
  }
  for (int j = lane; j < A; j += 32) dst[L.action + j] = state_absorbing ? 0.f : action[j];
  if (lane == 0) {
    dst[L.reward] = reward;
    dst[L.terminal] = terminal;
    dst[L.timeout] = timeout;
    dst[L.weight] = 1.f;  // memory.py:41
    dst[L.step] = step;
    for (int j = L.step + 1; j < L.len; ++j) dst[j] = 0.f;
  }
}

// One warp per replica.
__global__ void replay_append_kernel(il_replay mem, int R, const float* __restrict__ step, const float* __restrict__ state, const float* __restrict__ action,
                                     const float* __restrict__ reward, const float* __restrict__ next_state, const float* __restrict__ terminal,
                                     const float* __restrict__ timeout, const int32_t* __restrict__ active, int wrap) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x & 31;
  if (r >= R) return;
  if (active && !active[r]) return;
  const int S = mem.S, A = mem.A;
  const RowLayout L = row_layout(S, A);
  const int mi = mem.shared ? 0 : r;
  float* rows = mem.rows + (int64_t)r * mem.replica_stride;
  int idx = mem.idx[mi];
  const float term = terminal[r], tout = timeout[r], stp = step[r];
  const bool do_wrap = wrap && term != 0.f;  // train.py:162
  // memory.py:40-44 (+ :67: when wrapping, the stored next state becomes the absorbing state and terminal is cleared)
  write_row(rows + (int64_t)idx * L.len, L, S, A, lane, state + (int64_t)r * S, action + (int64_t)r * A, reward[r], next_state + (int64_t)r * S, do_wrap ? 0.f : term, tout,
            stp, false, do_wrap);
  int full = mem.full[mi];
  idx = (idx + 1) % mem.size;
  full = full || idx == 0;
  if (do_wrap) {  // memory.py:68: absorbing -> absorbing transition, zero action, zero reward, same step
    write_row(rows + (int64_t)idx * L.len, L, S, A, lane, nullptr, nullptr, 0.f, nullptr, 0.f, 0.f, stp, true, true);
    idx = (idx + 1) % mem.size;
    full = full || idx == 0;
  }
  __syncwarp();
  if (lane == 0) {
    mem.idx[mi] = idx;
    mem.full[mi] = full;
    if (term != 0.f || tout != 0.f) mem.num_trajectories[mi] += 1;
  }
}

// memory.py:65-68 as a separate call (wrap_for_absorbing_states on the row appended last). One warp per replica.
__global__ void replay_wrap_kernel(il_replay mem, int R, const int32_t* __restrict__ mask) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x & 31;
  if (r >= R) return;
  if (mask && !mask[r]) return;
  const int S = mem.S, A = mem.A;
  const RowLayout L = row_layout(S, A);
  const int mi = mem.shared ? 0 : r;
  float* rows = mem.rows + (int64_t)r * mem.replica_stride;
  int idx = mem.idx[mi];
  const int last = (idx - 1 + mem.size) % mem.size;
  float* lr = rows + (int64_t)last * L.len;
  for (int j = lane; j < S; j += 32) lr[L.next_state + j] = j == S - 1 ? 1.f : 0.f;
  const float stp = lr[L.step];
  __syncwarp();
  if (lane == 0) lr[L.terminal] = 0.f;
  write_row(rows + (int64_t)idx * L.len, L, S, A, lane, nullptr, nullptr, 0.f, nullptr, 0.f, 0.f, stp, true, true);
  __syncwarp();
  if (lane == 0) {
    idx = (idx + 1) % mem.size;
    mem.idx[mi] = idx;
    mem.full[mi] = mem.full[mi] || idx == 0;
  }
}

// memory.py:51-59: uniform over [0, size) (full) or [0, idx-1) (not full), never the newest row (idx-1) % size.
// seed_r (per-replica keys): blockIdx.y is the replica r, and its index k of n draws key seed_r[r] at counter (*counter + k), as a call over
// that replica alone would; NULL = one key `seed`, index i of all R * n at counter (*counter + i).
__global__ void replay_sample_idx_kernel(il_replay mem, int R, int n, int32_t* __restrict__ out, const float* __restrict__ uniform, uint64_t seed, uint64_t stream_id,
                                         const uint64_t* __restrict__ counter, const uint64_t* __restrict__ seed_r) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, k = i;
  int r;
  if (seed_r) {
    if (k >= n) return;
    r = (int)blockIdx.y;
    seed = seed_r[r];
    i = (int64_t)r * n + k;
  } else {
    if (i >= (int64_t)R * n) return;
    r = (int)(i / n);
  }
  const int mi = mem.shared ? 0 : r;
  const int idx = mem.idx[mi], full = mem.full[mi];
  uint32_t bits;
  if (uniform) {  // host-drawn U[0,1) (the reference draws on the host: memory.py:54)
    const float u = fminf(fmaxf(uniform[i], 0.f), 0.99999994f);
    bits = (uint32_t)(u * 4294967296.f);
  } else {
    const uint64_t c = (counter ? *counter : 0ull) + (uint64_t)k;
    bits = philox4x32_10(make_uint4((uint32_t)c, (uint32_t)(c >> 32), (uint32_t)stream_id, (uint32_t)(stream_id >> 32)), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32))).x;
  }
  int j;
  if (full) {
    const int newest = (idx - 1 + mem.size) % mem.size;
    j = (int)(((uint64_t)bits * (uint64_t)(mem.size - 1)) >> 32);
    if (j >= newest) j += 1;
  } else {
    const int count = idx - 1 > 0 ? idx - 1 : 1;
    j = (int)(((uint64_t)bits * (uint64_t)count) >> 32);
  }
  out[i] = j;
}

// one thread per float4 of the output
__global__ void replay_gather_kernel(const float* __restrict__ rows, int64_t mem_rs, int size, int row4, const int32_t* __restrict__ idx, float* __restrict__ out, int64_t out_rs,
                                     int R, int B) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)R * B * row4) return;
  const int q = (int)(t % row4);
  const int64_t rowi = t / row4;
  const int r = (int)(rowi / B), b = (int)(rowi % B);
  int src = idx[rowi];
  src = src < 0 ? 0 : (src >= size ? size - 1 : src);
  const float4 v = __ldg(reinterpret_cast<const float4*>(rows + (int64_t)r * mem_rs + (int64_t)src * row4 * 4) + q);
  reinterpret_cast<float4*>(out + (int64_t)r * out_rs + (int64_t)b * row4 * 4)[q] = v;
}

__global__ void mix_rows_kernel(float* __restrict__ dst, int64_t dst_rs, const float* __restrict__ src, int64_t src_rs, int row4, int half, int R) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)R * half * row4) return;
  const int q = (int)(t % row4);
  const int64_t rowi = t / row4;
  const int r = (int)(rowi / half), b = (int)(rowi % half);
  reinterpret_cast<float4*>(dst + (int64_t)r * dst_rs + (int64_t)b * row4 * 4)[q] = __ldg(reinterpret_cast<const float4*>(src + (int64_t)r * src_rs + (int64_t)b * row4 * 4) + q);
}

// transfer_transitions (memory.py:46-48): every row of `src` (a single-store memory) appended in order to every replica's
// ring: row (idx0 + i) % size <- src row i with weight 1 (append resets it, memory.py:41). One thread per float4 of a
// destination row; rows that a later row of the same transfer would overwrite (n > size) are skipped.
__global__ void replay_transfer_rows_kernel(il_replay dst, int R, const float* __restrict__ src_rows, int n, int row4) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)R * n * row4) return;
  const int q = (int)(t % row4);
  const int64_t ri = t / row4;
  const int r = (int)(ri / n), i = (int)(ri % n);
  if (i < n - dst.size) return;
  const int idx0 = dst.idx[dst.shared ? 0 : r];
  const RowLayout L = row_layout(dst.S, dst.A);
  float4 v = __ldg(reinterpret_cast<const float4*>(src_rows + (int64_t)i * row4 * 4) + q);
  if (L.weight / 4 == q) reinterpret_cast<float*>(&v)[L.weight % 4] = 1.f;
  reinterpret_cast<float4*>(dst.rows + (int64_t)r * dst.replica_stride + (int64_t)((idx0 + i) % dst.size) * row4 * 4)[q] = v;
}
// ring state after the rows above: idx, full, num_trajectories (+1 per terminal / timeout row, memory.py:44). One block per replica.
__global__ void replay_transfer_state_kernel(il_replay dst, const float* __restrict__ src_rows, int n) {
  __shared__ float red[32];
  const int r = blockIdx.x, mi = dst.shared ? 0 : r;
  const RowLayout L = row_layout(dst.S, dst.A);
  float ends = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float* row = src_rows + (int64_t)i * L.len;
    ends += (row[L.terminal] != 0.f || row[L.timeout] != 0.f) ? 1.f : 0.f;
  }
  ends = block_sum(ends, red);
  if (threadIdx.x == 0) {
    const int idx0 = dst.idx[mi];
    dst.idx[mi] = (int)(((int64_t)idx0 + n) % dst.size);
    dst.full[mi] = dst.full[mi] || ((int64_t)idx0 + n >= dst.size);
    dst.num_trajectories[mi] += (int)ends;
  }
}

// RewardRelabeller.resample_and_relabel (models.py:297-318), AdRIL (update_freq > 0) / SQIL (update_freq == 0). One thread per float4 of a row.
//   balanced: the whole batch is the expert batch on "expert" calls (flag[0] != 0) and the policy batch otherwise; the flag alternates per call.
//   unbalanced: the first B / 2 rows become expert rows (mix_expert_agent_transitions).
//   rewards: expert rows 1 / num_expert_trajectories (AdRIL) or 1 (SQIL); policy rows -1[round(step) > round(row step)] / max(num_trajectories, 1) or 0.
// update_freq_r / balanced_r ([R], optional): replica r runs as a uniform call with its own values; NULL = the scalar for every replica.
__global__ void adril_relabel_kernel(float* __restrict__ rows, int64_t rs, const float* __restrict__ ex, int64_t ex_rs, int R, int B, int row4, int off_reward, int off_step,
                                     int balanced, int update_freq, const int32_t* __restrict__ flag, const float* __restrict__ step_f, float step_offset,
                                     const int32_t* __restrict__ num_traj, int traj_shared, int num_expert_traj, const int32_t* __restrict__ update_freq_r,
                                     const int32_t* __restrict__ balanced_r) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)R * B * row4) return;
  const int q = (int)(t % row4);
  const int64_t rb = t / row4;
  const int r = (int)(rb / B), b = (int)(rb % B);
  if (update_freq_r) update_freq = update_freq_r[r];
  if (balanced_r) balanced = balanced_r[r];
  const bool expert_row = balanced ? (flag[0] != 0) : (b < B / 2);
  float4* dst = reinterpret_cast<float4*>(rows + (int64_t)r * rs + (int64_t)b * row4 * 4) + q;
  float4 v = expert_row ? __ldg(reinterpret_cast<const float4*>(ex + (int64_t)r * ex_rs + (int64_t)b * row4 * 4) + q) : *dst;
  if (off_reward / 4 == q) {
    float rew;
    if (expert_row) rew = update_freq > 0 ? 1.f / (float)num_expert_traj : 1.f;
    else if (update_freq > 0) {
      const float* rp = expert_row ? nullptr : rows + (int64_t)r * rs + (int64_t)b * row4 * 4;
      const float round_num = ceilf((step_f[r] + step_offset) / (float)update_freq);        // ceil(step / update_freq), models.py:313
      const float row_round = ceilf(rp[off_step] / (float)update_freq);                       // torch.ceil(transitions['step'] / update_freq)
      const int nt = num_traj[traj_shared ? 0 : r];
      rew = -1.f * (round_num > row_round ? 1.f : 0.f) / (float)(nt > 1 ? nt : 1);
    } else rew = 0.f;
    reinterpret_cast<float*>(&v)[off_reward % 4] = rew;
  }
  if (expert_row || off_reward / 4 == q) *dst = v;
}
__global__ void flag_toggle_kernel(int32_t* flag) { flag[0] = flag[0] ? 0 : 1; }

int check_replay(const il_replay* m, const char* what) {
  IL_CHECK(m && m->rows && m->idx && m->full && m->num_trajectories, "%s: null replay field", what);
  IL_CHECK(m->size > 0 && m->S > 0 && m->A > 0, "%s: size=%d S=%d A=%d", what, m->size, m->S, m->A);
  IL_CHECK(m->row == row_layout(m->S, m->A).len, "%s: row length %d != %d", what, m->row, row_layout(m->S, m->A).len);
  IL_CHECK((reinterpret_cast<uintptr_t>(m->rows) & 15) == 0 && m->replica_stride % 4 == 0, "%s: rows not 16-byte aligned", what);
  return 0;
}
int check_batch(const il_batch* b, const char* what) {
  IL_CHECK(b && b->rows, "%s: null batch", what);
  IL_CHECK(b->B > 0 && b->row == row_layout(b->S, b->A).len, "%s: B=%d row=%d (S=%d A=%d)", what, b->B, b->row, b->S, b->A);
  IL_CHECK((reinterpret_cast<uintptr_t>(b->rows) & 15) == 0 && b->replica_stride % 4 == 0, "%s: rows not 16-byte aligned", what);
  return 0;
}

}  // namespace

extern "C" int il_replay_append(il_handle* h, const il_replay* mem, int R, const float* step, const float* state, const float* action, const float* reward,
                                const float* next_state, const float* terminal, const float* timeout, const int32_t* active, int wrap, void* stream) {
  IL_CHECK(h, "il_replay_append: null handle");
  IL_TRY(check_replay(mem, "il_replay_append"));
  IL_CHECK(step && state && action && reward && next_state && terminal && timeout && R > 0, "il_replay_append: null input");
  IL_CHECK(!(wrap && mem->size < 2), "il_replay_append: absorbing wrap needs size >= 2");
  IL_LAUNCH(h, replay_append_kernel, (unsigned)((R * 32 + 127) / 128), 128, 0, (cudaStream_t)stream, *mem, R, step, state, action, reward, next_state, terminal, timeout, active,
            wrap);
  return 0;
}

extern "C" int il_replay_transfer(il_handle* h, const il_replay* dst, int R, const il_replay* src, void* stream) {
  IL_CHECK(h && R > 0, "il_replay_transfer: bad argument");
  IL_TRY(check_replay(dst, "il_replay_transfer(dst)"));
  IL_TRY(check_replay(src, "il_replay_transfer(src)"));
  IL_CHECK(dst->row == src->row && dst->S == src->S && dst->A == src->A, "il_replay_transfer: row layout mismatch");
  IL_CHECK(!dst->shared || R == 1, "il_replay_transfer: a shared destination takes one writer");
  const int n = src->size, row4 = src->row / 4;  // a pre-filled memory holds `size` valid rows (memory.py:18-23, __len__ :37-38)
  const int64_t total = (int64_t)R * n * row4;
  IL_LAUNCH(h, replay_transfer_rows_kernel, (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream, *dst, R, src->rows, n, row4);
  IL_LAUNCH(h, replay_transfer_state_kernel, (unsigned)(dst->shared ? 1 : R), 256, 0, (cudaStream_t)stream, *dst, src->rows, n);
  return 0;
}

extern "C" int il_replay_wrap_absorbing(il_handle* h, const il_replay* mem, int R, const int32_t* mask, void* stream) {
  IL_CHECK(h && R > 0, "il_replay_wrap_absorbing: bad argument");
  IL_TRY(check_replay(mem, "il_replay_wrap_absorbing"));
  IL_CHECK(mem->size >= 2, "il_replay_wrap_absorbing: size must be >= 2");
  IL_LAUNCH(h, replay_wrap_kernel, (unsigned)((R * 32 + 127) / 128), 128, 0, (cudaStream_t)stream, *mem, R, mask);
  return 0;
}

extern "C" int il_replay_sample_indices(il_handle* h, const il_replay* mem, int R, int n, int32_t* idx_out, const float* uniform, uint64_t seed, uint64_t stream_id,
                                        const uint64_t* counter, void* stream) {
  IL_CHECK(h && idx_out && R > 0 && n > 0, "il_replay_sample_indices: bad argument");
  IL_TRY(check_replay(mem, "il_replay_sample_indices"));
  IL_LAUNCH(h, replay_sample_idx_kernel, (unsigned)(((int64_t)R * n + 255) / 256), 256, 0, (cudaStream_t)stream, *mem, R, n, idx_out, uniform, seed, stream_id, counter,
            nullptr);
  return 0;
}

extern "C" int il_replay_sample_indices_r(il_handle* h, const il_replay* mem, int R, int n, int32_t* idx_out, const float* uniform, const uint64_t* seed_r,
                                          uint64_t stream_id, const uint64_t* counter, void* stream) {
  IL_CHECK(h && idx_out && seed_r && R > 0 && R <= IL_MAX_GRID_Y && n > 0, "il_replay_sample_indices_r: bad argument (R = %d)", R);
  IL_TRY(check_replay(mem, "il_replay_sample_indices_r"));
  IL_LAUNCH(h, replay_sample_idx_kernel, dim3((unsigned)((n + 255) / 256), (unsigned)R), 256, 0, (cudaStream_t)stream, *mem, R, n, idx_out, uniform, 0ull, stream_id,
            counter, seed_r);
  return 0;
}

extern "C" int il_replay_gather(il_handle* h, const il_replay* mem, int R, const int32_t* idx, const il_batch* out, void* stream) {
  IL_CHECK(h && idx && R > 0, "il_replay_gather: bad argument");
  IL_TRY(check_replay(mem, "il_replay_gather"));
  IL_TRY(check_batch(out, "il_replay_gather"));
  IL_CHECK(out->row == mem->row && out->S == mem->S && out->A == mem->A, "il_replay_gather: batch/replay shape mismatch");
  const int row4 = mem->row / 4;
  const int64_t total = (int64_t)R * out->B * row4;
  IL_LAUNCH(h, replay_gather_kernel, (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream, mem->rows, mem->replica_stride, mem->size, row4, idx, out->rows,
            out->replica_stride, R, out->B);
  return 0;
}

// With update_freq_r / balanced_r the scalars keep a host-known meaning (the host cannot read device arrays during graph capture): balanced = 1
// when any replica is balanced, update_freq = the largest value. The alternation flag stays one device scalar: every replica of a program
// calls the relabeller at the same steps, so the balanced replicas see the flag sequence of a uniform balanced run and the others never read it.
extern "C" int il_adril_relabel(il_handle* h, const il_batch* batch, const il_batch* expert, int R, int balanced, int update_freq, int32_t* sample_expert_flag,
                                const float* step_f, float step_offset, const int32_t* num_trajectories, int trajectories_shared, int num_expert_trajectories, void* stream,
                                const int32_t* update_freq_r, const int32_t* balanced_r) {
  IL_CHECK(h && R > 0, "il_adril_relabel: bad argument");
  IL_TRY(check_batch(batch, "il_adril_relabel(batch)"));
  IL_TRY(check_batch(expert, "il_adril_relabel(expert)"));
  IL_CHECK(batch->row == expert->row && expert->B >= (balanced ? batch->B : batch->B / 2), "il_adril_relabel: shape mismatch");
  IL_CHECK(!balanced || sample_expert_flag, "il_adril_relabel: balanced sampling needs the alternation flag");
  IL_CHECK(update_freq == 0 || (step_f && num_trajectories && num_expert_trajectories > 0), "il_adril_relabel: AdRIL relabelling needs step / trajectory counters");
  const RowLayout L = row_layout(batch->S, batch->A);
  const int row4 = batch->row / 4;
  const int64_t total = (int64_t)R * batch->B * row4;
  IL_LAUNCH(h, adril_relabel_kernel, (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream, batch->rows, batch->replica_stride, expert->rows, expert->replica_stride, R, batch->B, row4,
            L.reward, L.step, balanced, update_freq, sample_expert_flag, step_f, step_offset, num_trajectories, trajectories_shared, num_expert_trajectories, update_freq_r,
            balanced_r);
  if (balanced) IL_LAUNCH(h, flag_toggle_kernel, 1, 1, 0, (cudaStream_t)stream, sample_expert_flag);
  return 0;
}

extern "C" int il_mix_expert_rows(il_handle* h, const il_batch* batch, const il_batch* expert, int R, void* stream) {
  IL_CHECK(h && R > 0, "il_mix_expert_rows: bad argument");
  IL_TRY(check_batch(batch, "il_mix_expert_rows(batch)"));
  IL_TRY(check_batch(expert, "il_mix_expert_rows(expert)"));
  IL_CHECK(batch->row == expert->row && expert->B >= batch->B / 2, "il_mix_expert_rows: shape mismatch");
  const int half = batch->B / 2, row4 = batch->row / 4;
  if (half == 0) return 0;
  const int64_t total = (int64_t)R * half * row4;
  IL_LAUNCH(h, mix_rows_kernel, (unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream, batch->rows, batch->replica_stride, expert->rows, expert->replica_stride, row4,
            half, R);
  return 0;
}
