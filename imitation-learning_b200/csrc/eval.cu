// evaluate_agent (evaluation.py:11-35) as ONE device program: R x episodes greedy episodes advance in lock-step inside a CUDA
// graph whose body (greedy actor forward -> env step + return accumulation) sits in a WHILE conditional node; the last block of
// every iteration sets the loop condition on the device (cudaGraphSetConditional), so the host launches once and is not involved
// again until every episode has ended. Finished episodes are frozen, which makes the lock-step batch the same computation as the
// reference's sequential batch-size-1 episodes (episodes are independent given their initial states).
//   il_eval_rollout : the rollout above (+ optional trajectory recording, evaluation.py:30-33)
//   il_return_allreduce : per-rank (sum, sum of squares, count) of the returns + ncclAllReduce on the same stream (train.py:213-219
//                         across the seed-sharded ranks, SURVEY §8e). NCCL is bound at run time (the copy torch already loaded).
#include <dlfcn.h>

#include "env.cuh"
#include "mlp.cuh"

// Up to 8 episodes per replica the whole actor runs in one weight-streaming kernel; above that (the reference's 30 evaluation episodes,
// conf/train_config.yaml:23) the per-layer grouped GEMM program is used: the single-kernel path is bound by its shared-memory operand
// loads.
constexpr int EVAL_SMALL_MAX = 8;

struct EvalCounters {  // device-resident loop state
  int32_t running;      // episodes still running after the current iteration (accumulated by the blocks of the step kernel)
  int32_t ticket;       // blocks that have finished the current iteration
  int32_t iterations;   // loop iterations executed
  int32_t _pad;
  int64_t env_steps;    // environment steps executed (sum over episodes)
};

namespace {

struct EvalStepParams {
  il_env env;
  int n;                 // R * episodes environments
  int act_E, act_EP;     // the action of environment e sits at row (e / act_E) * act_EP + e % act_E (padded rows per replica on the tensor-core path; E == EP otherwise)
  const float* action;   // [n, act]
  float* state;          // [n, S]: read by the actor, overwritten with the next state
  float* returns;        // [n]
  int32_t* finished;     // [n]
  EvalCounters* ctr;
  cudaGraphConditionalHandle cond;
  int max_iterations;
  // trajectories (evaluation.py:22-23,30-33), optional
  float* traj_states;    // [n, T, S]
  float* traj_actions;   // [n, T, act]
  float* traj_rewards;   // [n, T]
  int32_t* traj_len;     // [n]
  int traj_T;
};

// one warp per environment (4 per block)
__global__ void __launch_bounds__(128) eval_step_kernel(const EvalStepParams p) {
  const int lane = threadIdx.x & 31, e = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int S = p.env.obs + (p.env.absorbing ? 1 : 0), act = p.env.act;
  int running = 0;
  if (e < p.n && !p.finished[e]) {
    const float* a = p.action + ((int64_t)(e / p.act_E) * p.act_EP + e % p.act_E) * act;
    float* st = p.state + (int64_t)e * S;
    const int t = p.env.t[e];
    const bool rec = p.traj_states != nullptr && t < p.traj_T;
    if (rec) {  // the (state, action) pair the step is taken from
      for (int j = lane; j < S; j += 32) p.traj_states[((int64_t)e * p.traj_T + t) * S + j] = st[j];
      for (int j = lane; j < act; j += 32) p.traj_actions[((int64_t)e * p.traj_T + t) * act + j] = a[j];
    }
    __syncwarp();
    const EnvStepOut o = env_step_core(p.env, e, lane, a, st);
    if (lane == 0) {
      p.returns[e] += o.reward;  // evaluation.py:24,28
      if (rec) { p.traj_rewards[(int64_t)e * p.traj_T + t] = o.reward; p.traj_len[e] = t + 1; }
      if (o.early || o.time_limit) p.finished[e] = 1;  // environments.py:38: gym's done (early termination or time limit)
      else running = 1;
    }
  }
  // loop control: per-block count -> global count; the last block of the iteration decides whether the body runs again
  __shared__ int s_run[4];
  if (lane == 0) s_run[threadIdx.x >> 5] = running;
  __syncthreads();
  if (threadIdx.x == 0) {
    const int r = s_run[0] + s_run[1] + s_run[2] + s_run[3];
    if (r) atomicAdd(&p.ctr->running, r);
    __threadfence();
    const int ticket = atomicAdd(&p.ctr->ticket, 1);
    if (ticket == (int)gridDim.x - 1) {
      __threadfence();
      const int still = atomicAdd(&p.ctr->running, 0);
      const int it = p.ctr->iterations + 1;
      p.ctr->iterations = it;
      p.ctr->env_steps += still;  // every running episode takes one more step next iteration (the first iteration's steps are added at reset)
      p.ctr->running = 0;
      p.ctr->ticket = 0;
      cudaGraphSetConditional(p.cond, (still > 0 && it < p.max_iterations) ? 1u : 0u);
    }
  }
}

// rows [E, EP) of every replica's input block stay zero: they only pad the row count of the grouped GEMMs to the tile height of the wgmma engine
__global__ void eval_pad_rows_kernel(const float* __restrict__ state, float* __restrict__ xpad, int R, int E, int EP, int S) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)R * E * S) return;
  const int64_t row = i / S;
  const int k = (int)(i % S);
  xpad[((row / E) * EP + row % E) * S + k] = state[i];
}

__global__ void eval_init_kernel(float* returns, int32_t* finished, int32_t* traj_len, EvalCounters* ctr, int n, float* xpad, int64_t xpad_n) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < xpad_n; j += (int64_t)gridDim.x * blockDim.x) xpad[j] = 0.f;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    returns[i] = 0.f;
    finished[i] = 0;
    if (traj_len) traj_len[i] = 0;
  }
  if (i == 0) { ctr->running = 0; ctr->ticket = 0; ctr->iterations = 0; ctr->env_steps = n; }
}

__global__ void eval_export_kernel(const EvalCounters* ctr, int64_t* out2) {
  out2[0] = ctr->iterations;
  out2[1] = ctr->env_steps;
}

__global__ void return_stats3_kernel(const float* __restrict__ returns, int64_t n, float* __restrict__ out3) {
  __shared__ float red[32];
  float s = 0.f, s2 = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = returns[i];
    s += v;
    s2 += v * v;
  }
  s = block_sum(s, red);
  s2 = block_sum(s2, red);
  if (threadIdx.x == 0) { out3[0] = s; out3[1] = s2; out3[2] = (float)n; }
}

struct EvalGraph {
  il_eval_args key;
  int ep;  // padded rows per replica the graph was built for (depends on the gemm mode of the handle)
  cudaGraph_t graph;
  cudaGraphExec_t exec;
};

void eval_graph_free(EvalGraph* g) {
  if (!g) return;
  if (g->exec) cudaGraphExecDestroy(g->exec);
  if (g->graph) cudaGraphDestroy(g->graph);
  delete g;
}

}  // namespace

void il_eval_release(il_handle* h) {
  eval_graph_free(static_cast<EvalGraph*>(h->eval_graph));
  h->eval_graph = nullptr;
}

// Builds  [reset] -> while (episodes running) { greedy actor forward ; env step + accumulate + loop condition }
// Rows per replica of the greedy forward: the episode count, or — when the grouped GEMM program is used and the tensor-core engine is on and
// applicable (256-wide hidden layers) — the next multiple of the 128-row wgmma tile.
static int eval_padded_rows(const il_handle* h, const il_eval_args* a) {
  const int E = a->episodes, L = a->actor.n_layers;
  if (E <= EVAL_SMALL_MAX || h->gemm_mode == IL_GEMM_FP32 || L < 2) return E;
  for (int l = 1; l < L; ++l)
    if (a->actor.dims[l] != 256) return E;
  return (E + 127) / 128 * 128;
}
static int eval_build_impl(il_handle* h, EvalGraph* eg, const il_eval_args* a, float* action, int32_t* finished, EvalCounters* ctr, char* ws, cudaStream_t st);
// Capturing records kernel nodes without running anything, so it happens on a private stream (the caller's stream may be the legacy
// default stream, which cannot capture); whatever goes wrong, that stream is taken out of capture mode again.
static int eval_build(il_handle* h, EvalGraph* eg, const il_eval_args* a, float* action, int32_t* finished, EvalCounters* ctr, char* ws) {
  if (!h->build_stream) IL_CUDA(cudaStreamCreateWithFlags(&h->build_stream, cudaStreamNonBlocking));
  const int rc = eval_build_impl(h, eg, a, action, finished, ctr, ws, h->build_stream);
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(h->build_stream, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone) {
    cudaGraph_t junk = nullptr;
    cudaStreamEndCapture(h->build_stream, &junk);
  }
  if (rc != 0) cudaGetLastError();
  return rc;
}
static int eval_build_impl(il_handle* h, EvalGraph* eg, const il_eval_args* a, float* action, int32_t* finished, EvalCounters* ctr, char* ws, cudaStream_t st) {
  const int R = a->R, E = a->episodes, act = a->env.act, S = a->env.obs + (a->env.absorbing ? 1 : 0), n = R * E;
  IL_CUDA(cudaGraphCreate(&eg->graph, 0));
  cudaGraphConditionalHandle cond;
  IL_CUDA(cudaGraphConditionalHandleCreate(&cond, eg->graph, 1, cudaGraphCondAssignDefault));
  // node 0: reset of returns / finished flags / counters, captured into the top-level graph
  IL_CUDA(cudaStreamBeginCaptureToGraph(st, eg->graph, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
  // E > 8 episodes per replica: the greedy forward is a grouped GEMM program; with the tensor-core engine on, the rows of every replica are padded to a
  // multiple of 128 (zero rows) so that the 256-wide layers run on wgmma tiles instead of the fp32 FFMA engine (30 rows -> 128: 4x the MMA work; the
  // loop body is bound by streaming every replica's weights once per step)
  const int EP = eval_padded_rows(h, a);
  float* xpad = nullptr;
  eval_init_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a->returns, finished, a->traj_len, ctr, n, EP != E ? reinterpret_cast<float*>(ws) : nullptr, EP != E ? (int64_t)R * EP * S : 0);
  h->launches++;
  cudaGraph_t captured = nullptr;
  IL_CUDA(cudaStreamEndCapture(st, &captured));
  size_t n_nodes = 0;
  IL_CUDA(cudaGraphGetNodes(eg->graph, nullptr, &n_nodes));
  IL_CHECK(n_nodes == 1, "il_eval_rollout: unexpected graph shape (%zu nodes)", n_nodes);
  cudaGraphNode_t init_node;
  IL_CUDA(cudaGraphGetNodes(eg->graph, &init_node, &n_nodes));
  // node 1: the while loop
  cudaGraphNodeParams np = {};
  np.type = cudaGraphNodeTypeConditional;
  np.conditional.handle = cond;
  np.conditional.type = cudaGraphCondTypeWhile;
  np.conditional.size = 1;
  cudaGraphNode_t while_node;
  IL_CUDA(cudaGraphAddNode(&while_node, eg->graph, &init_node, 1, &np));
  cudaGraph_t body = np.conditional.phGraph_out[0];
  IL_CUDA(cudaStreamBeginCaptureToGraph(st, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
  int rc = 0;
  {  // evaluation.py:21: greedy action for every episode (frozen ones ignore theirs)
    const MatView X{a->state, (int64_t)E * S, 1, S};
    if (E <= EVAL_SMALL_MAX) {
      rc = mlp_small_forward(h, &a->actor, R, E, X, action, st, act);
    } else {
      char* w1 = ws;
      MatView Xin = X;
      if (EP != E) {
        xpad = reinterpret_cast<float*>(ws);
        w1 = ws + il_align_up((int64_t)R * EP * S * 4, 256);
        eval_pad_rows_kernel<<<(unsigned)(((int64_t)n * S + 255) / 256), 256, 0, st>>>(a->state, xpad, R, E, EP, S);
        h->launches++;
        Xin = MatView{xpad, (int64_t)EP * S, 1, S};
      }
      MlpActs acts;
      char* w2 = mlp_acts_carve(&a->actor, R, EP, w1, &acts);
      float* head = reinterpret_cast<float*>(w2);
      rc = mlp_forward(h, &a->actor, R, EP, Xin, acts, head, (int64_t)EP * 2 * act, 2 * act, st, MLP_KEEP_NONE);
      if (rc == 0) {
        HeadFwdArgs ha{};
        ha.head = head; ha.action = action; ha.action_rs = (int64_t)EP * act; ha.ld_action = act; ha.R = R; ha.n = EP; ha.A = act;
        rc = launch_actor_head(h, ha, st);
      }
    }
  }
  if (rc == 0) {
    EvalStepParams sp{};
    sp.env = a->env; sp.n = n; sp.act_E = E; sp.act_EP = (E > EVAL_SMALL_MAX) ? EP : E; sp.action = action; sp.state = a->state; sp.returns = a->returns; sp.finished = finished; sp.ctr = ctr; sp.cond = cond;
    sp.max_iterations = a->max_steps;
    sp.traj_states = a->traj_states; sp.traj_actions = a->traj_actions; sp.traj_rewards = a->traj_rewards; sp.traj_len = a->traj_len; sp.traj_T = a->traj_T;
    eval_step_kernel<<<(unsigned)((n + 3) / 4), 128, 0, st>>>(sp);
    h->launches++;
  }
  cudaGraph_t body_out = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(st, &body_out);  // always leave capture mode, also on errors above
  if (rc != 0) return rc;
  IL_CHECK(ce == cudaSuccess, "il_eval_rollout: capture of the loop body failed: %s", cudaGetErrorString(ce));
  IL_CUDA(cudaGraphInstantiate(&eg->exec, eg->graph, 0));
  return 0;
}

extern "C" int64_t il_eval_workspace_bytes(const il_eval_args* a) {
  if (!a || a->R <= 0 || a->episodes <= 0) return -1;
  const int64_t n = (int64_t)a->R * a->episodes;
  const int act = a->env.act;
  // action [n, act] | finished [n] | counters | (episodes > 32: per-layer activations + head of the general MLP path)
  // worst case over the gemm modes: rows padded to 128 per replica (tensor-core path)
  const int64_t EP = (a->episodes + 127) / 128 * 128, np = (int64_t)a->R * EP;
  int64_t b = il_align_up(np * act * 4, 256) + il_align_up(n * 4, 256) + 256;
  if (a->episodes > EVAL_SMALL_MAX)
    b += il_align_up(np * a->actor.dims[0] * 4, 256) + mlp_acts_bytes(&a->actor, a->R, (int)EP) + il_align_up(np * a->actor.dims[a->actor.n_layers] * 4, 256);
  return b;
}

extern "C" int il_eval_rollout(il_handle* h, const il_eval_args* a, void* stream) {
  IL_CHECK(h && a, "il_eval_rollout: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  IL_TRY(mlp_validate(&a->actor, "il_eval_rollout(actor)"));
  const int R = a->R, E = a->episodes, act = a->env.act, S = a->env.obs + (a->env.absorbing ? 1 : 0);
  IL_CHECK(R > 0 && E > 0 && a->state && a->returns && a->workspace && a->max_steps > 0, "il_eval_rollout: bad argument");
  IL_CHECK(a->env.M && a->env.N && a->env.c && a->env.w_r && a->env.x && a->env.t && a->env.obs > 0 && a->env.obs <= 32 * MAX_OBS_PER_LANE, "il_eval_rollout: bad env");
  IL_CHECK(a->actor.dims[0] == S && a->actor.dims[a->actor.n_layers] == 2 * act, "il_eval_rollout: actor dims do not match the environment (S=%d, A=%d)", S, act);
  IL_CHECK(a->workspace_bytes >= il_eval_workspace_bytes(a), "il_eval_rollout: workspace too small");
  IL_CHECK(!a->traj_states || (a->traj_actions && a->traj_rewards && a->traj_len && a->traj_T > 0), "il_eval_rollout: incomplete trajectory buffers");
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  IL_CUDA(cudaStreamIsCapturing(st, &cs));
  IL_CHECK(cs == cudaStreamCaptureStatusNone, "il_eval_rollout: cannot run inside a stream capture (a graph with a conditional node cannot be a child graph)");
  const int n = R * E;
  char* ws = static_cast<char*>(a->workspace);
  float* action = reinterpret_cast<float*>(ws); ws += il_align_up((int64_t)R * ((E + 127) / 128 * 128) * act * 4, 256);  // sized for the padded layout (il_eval_workspace_bytes)
  int32_t* finished = reinterpret_cast<int32_t*>(ws); ws += il_align_up((int64_t)n * 4, 256);
  EvalCounters* ctr = reinterpret_cast<EvalCounters*>(ws); ws += 256;

  EvalGraph* eg = static_cast<EvalGraph*>(h->eval_graph);
  if (eg && (memcmp(&eg->key, a, sizeof(il_eval_args)) != 0 || eg->ep != eval_padded_rows(h, a))) {  // different buffers / shapes: rebuild (the old graph may still be running on this stream)
    IL_CUDA(cudaStreamSynchronize(st));
    il_eval_release(h);
    eg = nullptr;
  }
  if (!eg) {
    eg = new EvalGraph();
    eg->key = *a; eg->graph = nullptr; eg->exec = nullptr; eg->ep = eval_padded_rows(h, a);
    h->eval_graph = eg;
    const int rc = eval_build(h, eg, a, action, finished, ctr, ws);
    if (rc != 0) { il_eval_release(h); return rc; }
  }
  IL_CUDA(cudaGraphLaunch(eg->exec, st));
  if (a->out_counters) IL_LAUNCH(h, eval_export_kernel, 1, 1, 0, st, ctr, a->out_counters);
  return 0;
}

// ---- NCCL bound at run time -------------------------------------------------------------------------------------------------
namespace {
struct NcclId { char b[128]; };  // ncclUniqueId (passed by value)
struct NcclApi {
  void* lib;
  int (*GetUniqueId)(void*);
  int (*CommInitRank)(void**, int, NcclId, int);
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t);
  int (*CommDestroy)(void*);
  const char* (*GetErrorString)(int);
};
NcclApi g_nccl = {};
typedef decltype(NcclApi::CommInitRank) InitFn;

int nccl_load() {
  if (g_nccl.lib) return 0;
  void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);  // the copy the host framework (torch) already mapped, if any
  if (!lib) lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  IL_CHECK(lib, "NCCL not found (libnccl.so.2): %s", dlerror());
  g_nccl.GetUniqueId = reinterpret_cast<int (*)(void*)>(dlsym(lib, "ncclGetUniqueId"));
  g_nccl.CommInitRank = reinterpret_cast<InitFn>(dlsym(lib, "ncclCommInitRank"));
  g_nccl.AllReduce = reinterpret_cast<int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t)>(dlsym(lib, "ncclAllReduce"));
  g_nccl.CommDestroy = reinterpret_cast<int (*)(void*)>(dlsym(lib, "ncclCommDestroy"));
  g_nccl.GetErrorString = reinterpret_cast<const char* (*)(int)>(dlsym(lib, "ncclGetErrorString"));
  IL_CHECK(g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.AllReduce && g_nccl.CommDestroy && g_nccl.GetErrorString, "NCCL symbols missing in libnccl.so.2");
  g_nccl.lib = lib;
  return 0;
}
#define IL_NCCL(expr)                                                                                  \
  do {                                                                                                 \
    int _r = (expr);                                                                                   \
    if (_r != 0) IL_FAIL("%s failed: %s", #expr, g_nccl.GetErrorString ? g_nccl.GetErrorString(_r) : "?"); \
  } while (0)
}  // namespace

extern "C" int il_nccl_unique_id(uint8_t* out128) {
  IL_CHECK(out128, "il_nccl_unique_id: null argument");
  IL_TRY(nccl_load());
  IL_NCCL(g_nccl.GetUniqueId(out128));
  return 0;
}

extern "C" int il_nccl_comm_create(const uint8_t* id128, int rank, int world, void** comm) {
  IL_CHECK(id128 && comm && world >= 1 && rank >= 0 && rank < world, "il_nccl_comm_create: bad argument");
  IL_TRY(nccl_load());
  NcclId id;
  memcpy(id.b, id128, 128);
  IL_NCCL(g_nccl.CommInitRank(comm, world, id, rank));
  return 0;
}

extern "C" int il_nccl_comm_destroy(void* comm) {
  if (!comm) return 0;
  IL_TRY(nccl_load());
  IL_NCCL(g_nccl.CommDestroy(comm));
  return 0;
}

extern "C" int il_return_allreduce(il_handle* h, void* nccl_comm, const float* returns, int64_t n, float* out3, void* stream) {
  IL_CHECK(h && returns && out3 && n > 0, "il_return_allreduce: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  IL_LAUNCH(h, return_stats3_kernel, 1, 1024, 0, st, returns, n, out3);
  if (nccl_comm) {
    IL_TRY(nccl_load());
    IL_NCCL(g_nccl.AllReduce(out3, out3, 3, /* ncclFloat32 */ 7, /* ncclSum */ 0, nccl_comm, st));
  }
  return 0;
}
