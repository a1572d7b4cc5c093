// agogo_b200 — host side of the engine: the C ABI of include/agogo_b200.h over the CUDA kernels.
// No CPU fallback: creation fails with AZ_ERR_CUDA when there is no usable CUDA device.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/agogo_b200.h"
#include "mcts_dev.cuh"
#include "nn.cuh"
#include "tower_tc.cuh"
#include "train.cuh"

#include <dlfcn.h>
#include <nccl.h>

// kernels (mcts.cu)
size_t mcts_ws_bytes(const GameP& P, int cellsP);
void mcts_set_smem_limits(const GameP& P, int cellsP);
void launch_arena_begin(const GameP& P, const EngineDev& E, int n_games, const int* coins, unsigned long long game_base, cudaStream_t s);
void launch_assign_slots(const GameP& P, const EngineDev& E, int n_games, cudaStream_t s);
void launch_search_begin(const GameP& P, const EngineDev& E, int n_games, cudaStream_t s);
void launch_encode_roots(const GameP& P, const EngineDev& E, int n_games, cudaStream_t s);
void launch_select(const GameP& P, const EngineDev& E, int n_games, cudaStream_t s);
void launch_infer_simple(const GameP& P, const EngineDev& E, int n_games, cudaStream_t s);
void launch_expand_backup(const GameP& P, const EngineDev& E, int n_games, cudaStream_t s);
void launch_search_end(const GameP& P, const EngineDev& E, int n_games, int record, cudaStream_t s);
void launch_rules_apply(const GameP& P, int cellsP, int n, const int* boards, const int* players, const int* moves,
                        int* check, int* applied, int* out_boards, int* taken, cudaStream_t s);
void launch_rules_status(const GameP& P, int cellsP, int n, const int* boards, const int* passes, int* ended, int* winner,
                         float* sb, float* sw, cudaStream_t s);

static thread_local std::string g_create_error;

static inline uint64_t splitmix64(uint64_t* s) {
  uint64_t z = (*s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
static inline uint64_t derive_seed(uint64_t seed, uint64_t stream) {
  uint64_t s = seed ^ (0xD1B54A32D192ED03ull * (stream + 1));
  return splitmix64(&s);
}

struct HostExample { std::vector<float> board, policy; float value; };
struct HostRecord { std::vector<int32_t> moves; int32_t winner = 0, a_player = 0, n_examples = 0; };

struct az_engine {
  az_engine_desc d;
  GameP P;
  EngineDev E;  // device pointers
  int device = 0;
  cudaStream_t stream = nullptr;
  std::vector<void*> allocs;
  std::vector<unsigned long long> zt64;  // host copy of the position keys (external states are hashed on the host)
  NetLayout L;
  float* net_params[2] = {nullptr, nullptr};  // train-form, device
  Snapshot snap[2];
  bool snap_valid[2] = {false, false};
  Fp32Scratch fp32;
  TcTower tc[2];
  bool use_tc = false;
  int inf_kind[2] = {-1, -1};
  float* table_dev[2] = {nullptr, nullptr};
  float* table_val_dev[2] = {nullptr, nullptr};
  int* coins_dev = nullptr;
  uint64_t coin_state = 0;
  uint64_t games_started = 0;  // per-tree RNG streams: tree t of the c-th game = stream 2c + t of the tree seed
  // play state
  bool in_play = false, record = false;
  int n_play = 0;
  std::vector<std::vector<HostExample>> ex_by_game;
  std::vector<HostExample> examples;
  std::vector<HostRecord> records;
  float wins[2] = {0, 0}, loss[2] = {0, 0}, draw[2] = {0, 0};
  unsigned long long launches = 0;
  // pinned staging
  float *h_ex_board = nullptr, *h_ex_policy = nullptr, *h_ex_value = nullptr;
  int32_t* h_ex_valid = nullptr;
  int32_t* h_small = nullptr;  // [n_active, err]
  // one MCTS wave (select -> evaluate -> expand/backup) captured as a CUDA graph: every kernel argument is
  // device-resident state, so the captured launch sequence is replayed for each of the `sims` waves
  cudaGraphExec_t wave_graph = nullptr;
  int wave_graph_n = -1;
  uint64_t wave_graph_version = 0, cfg_version = 1;
  unsigned long long wave_graph_launches = 0;
  bool graphs_enabled = true, profiling = false, prof_region = false;
  int32_t* round_workers_dev = nullptr;  // mcts.Config workers: how many the current round starts
  int round_workers_host = -1;
  cudaEvent_t prof_start = nullptr, prof_stop = nullptr;  // region timing between az_profile(1) and az_profile(0)
  TrainWS train;
  void* comm = nullptr;  // ncclComm_t (bootstrap of the peer-memory path; plain all-reduce as the checked alternative)
  int rank = 0, world = 1;
  // peer-memory collective (K8): IPC-mapped gradient / parameter / flag buffers of every rank
  bool p2p = false;
  std::vector<void*> ipc_opened;
  float** d_peer_grads = nullptr;
  float** d_peer_params[2] = {nullptr, nullptr};
  int** d_peer_flags = nullptr;
  int* my_flags = nullptr;
  unsigned int* done_counter = nullptr;
  int epoch = 0, num_sms = 132;
  int32_t* d_agree = nullptr;  // step-count agreement of the data-parallel ranks (az_train)
  // Agent.Search on external positions: the position each agent's tree (game slot 0) was last searched on = t.prev
  struct ExtPrev { bool valid = false; int move_number = 0; std::vector<uint8_t> board; } ext_prev[2];
  mutable std::string err;

  template <class T>
  T* dalloc(size_t n, bool zero = true) {
    void* p = nullptr;
    CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)));
    if (zero) CUDA_CHECK(cudaMemset(p, 0, std::max<size_t>(n, 1) * sizeof(T)));
    allocs.push_back(p);
    return (T*)p;
  }
};

// NCCL is bound lazily with dlopen so that single-GPU use has no libnccl dependency at load time
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*);
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t);
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
  ncclResult_t (*CommDestroy)(ncclComm_t);
  const char* (*GetErrorString)(ncclResult_t);
};
static NcclApi& nccl_api() {
  static NcclApi api;
  static bool ok = false;
  if (!ok) {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) throw std::runtime_error(std::string("libnccl.so.2 not found: ") + dlerror());
    api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(h, "ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))dlsym(h, "ncclCommInitRank");
    api.AllReduce = (decltype(api.AllReduce))dlsym(h, "ncclAllReduce");
    api.AllGather = (decltype(api.AllGather))dlsym(h, "ncclAllGather");
    api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
    api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
    if (!api.GetUniqueId || !api.CommInitRank || !api.AllReduce || !api.AllGather || !api.CommDestroy || !api.GetErrorString)
      throw std::runtime_error("libnccl.so.2: missing symbols");
    ok = true;
  }
  return api;
}
static void nccl_allreduce_sum(az_engine* e, float* buf, size_t n) {
  NcclApi& a = nccl_api();
  ncclResult_t r = a.AllReduce(buf, buf, n, ncclFloat32, ncclSum, (ncclComm_t)e->comm, e->stream);
  if (r != ncclSuccess) throw std::runtime_error(std::string("ncclAllReduce: ") + a.GetErrorString(r));
}

#define GUARD_BEGIN try {
#define GUARD_END(e)                                                   \
  }                                                                    \
  catch (const CudaError& ce) { (e)->err = ce.msg; return AZ_ERR_CUDA; } \
  catch (const std::exception& ex) { (e)->err = ex.what(); return AZ_ERR_PANIC; }
// entry points that run inside an arena / search: any failure also leaves the "in play" state, so that the next call
// reports its own error instead of "during a running arena"
#define PLAY_ABORT(e) do { (e)->in_play = false; (e)->ex_by_game.clear(); } while (0)
#define GUARD_END_PLAY(e)                                                                  \
  }                                                                                        \
  catch (const CudaError& ce) { (e)->err = ce.msg; PLAY_ABORT(e); return AZ_ERR_CUDA; }     \
  catch (const std::exception& ex) { (e)->err = ex.what(); PLAY_ABORT(e); return AZ_ERR_PANIC; }

static int device_error_to_rc(az_engine* e, int bits) {
  if (!bits) return AZ_OK;
  std::string m = "device error:";
  if (bits & ERR_NO_ACTIVE_CHILD) m += " Cannot return nil (node.go:232: no selectable child)";
  if (bits & ERR_POOL_EXHAUSTED) m += " node pool exhausted (raise max_nodes_per_tree)";
  if (bits & ERR_ROOT_NO_CHILDREN) m += " root without children (search.go:141-149 fallback not implemented)";
  if (bits & ERR_ACT_OVERFLOW) m += " fp16 activation overflow in the tensor-core tower (lower act_scale_log2)";
  if (bits & ERR_NAN_PRIOR) m += " NaN prior";
  if (bits & ERR_PATH_OVERFLOW) m += " per-game move capacity exceeded (set game.max_moves)";
  if (bits & ERR_RESIGN_APPLIED) m += " index out of range (Arena applied Resign: State.Apply indexes board[-2])";
  if (bits & ERR_COMM_TIMEOUT) m += " gradient all-reduce: a peer rank never arrived (rank died, different batch count, or the call was not collective)";
  e->err = m;
  return AZ_ERR_PANIC;
}

extern "C" {

const char* az_build_info(void) { return "agogo_b200 0.1 sm_90a (hand-written CUDA; wgmma/TMA tower; no CPU fallback)"; }
const char* az_last_error(const az_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

void az_engine_destroy(az_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  if (e->comm && e->p2p) {  // peers have this rank's gradient / parameter / flag buffers IPC-mapped: nobody frees before everybody is done
    try {
      if (!e->d_agree) e->d_agree = e->dalloc<int32_t>(2);
      int32_t* d1 = e->d_agree;
      nccl_api().AllReduce(d1, d1, 1, ncclInt32, ncclSum, (ncclComm_t)e->comm, e->stream);
      cudaStreamSynchronize(e->stream);
    } catch (...) {}
  }
  for (void* p : e->ipc_opened) cudaIpcCloseMemHandle(p);
  e->ipc_opened.clear();
  for (void* p : e->allocs) cudaFree(p);
  for (int a = 0; a < 2; a++) { tc_tower_free(e->tc[a]); }
  train_ws_free(e->train);
  if (e->wave_graph) cudaGraphExecDestroy(e->wave_graph);
  if (e->prof_start) { cudaEventDestroy(e->prof_start); cudaEventDestroy(e->prof_stop); }
  for (void* p : e->ipc_opened) cudaIpcCloseMemHandle(p);
  if (e->comm) { try { nccl_api().CommDestroy((ncclComm_t)e->comm); } catch (...) {} }
  fp32_scratch_free(e->fp32);
  if (e->h_ex_board) cudaFreeHost(e->h_ex_board);
  if (e->h_ex_policy) cudaFreeHost(e->h_ex_policy);
  if (e->h_ex_value) cudaFreeHost(e->h_ex_value);
  if (e->h_ex_valid) cudaFreeHost(e->h_ex_valid);
  if (e->h_small) cudaFreeHost(e->h_small);
  if (e->stream) cudaStreamDestroy(e->stream);
  delete e;
}

int az_engine_create(const az_engine_desc* desc, az_engine** out) {
  if (!desc || !out) { g_create_error = "null argument"; return AZ_ERR_INVALID; }
  const az_dual_config& n = desc->nn;
  const az_mcts_config& m = desc->mcts;
  // dual.Config.IsValid (config.go:33-42) / mcts.Config.IsValid (tree.go:43-45): the reference panics
  if (!(n.k >= 1 && n.action_space >= 3 && n.shared_layers >= 0 && n.fc > 1 && n.batch_size >= 1 && n.features > 0)) {
    g_create_error = "NNConf is not valid. Unable to proceed"; return AZ_ERR_INVALID;
  }
  if (!(m.puct > 0 && m.puct <= 1)) { g_create_error = "MCTSConf is not valid. Unable to proceed"; return AZ_ERR_INVALID; }
  const az_game_desc& gd = desc->game;
  if (gd.kind < 0 || gd.kind > 2 || gd.m < 1 || gd.n < 1 || desc->n_games < 1) { g_create_error = "invalid game/n_games"; return AZ_ERR_INVALID; }
  if (gd.kind == AZ_GAME_WQ && gd.m != gd.n) { g_create_error = "wq boards are square"; return AZ_ERR_INVALID; }
  if (desc->encoder == AZ_ENC_WQ18 && gd.kind != AZ_GAME_WQ) { g_create_error = "WQEncoder needs State.Historical, which only wq provides on clones"; return AZ_ERR_UNSUPPORTED; }
  if (m.random_count > 0 && !(m.random_temperature > 0)) { g_create_error = "RandomCount > 0 needs RandomTemperature > 0"; return AZ_ERR_INVALID; }
  if (n.width != gd.n || n.height != gd.m) { g_create_error = "nn width/height must match the board"; return AZ_ERR_INVALID; }
  {  // expandAndSimulate reads policy[i] for i < ActionSpace and policy[len-1] (search.go:285-296): a narrower net panics
    const int A = gd.kind == AZ_GAME_C4 ? gd.n : gd.m * gd.n;
    if (n.action_space < A) { g_create_error = "index out of range: dual.Config.ActionSpace is smaller than the game's ActionSpace()"; return AZ_ERR_INVALID; }
  }
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev <= desc->device) {
    g_create_error = std::string("no usable CUDA device (") + cudaGetErrorString(ce) + "); agogo_b200 has no CPU fallback";
    return AZ_ERR_CUDA;
  }
  std::unique_ptr<az_engine> e(new az_engine);
  try {
    e->d = *desc;
    e->device = desc->device;
    CUDA_CHECK(cudaSetDevice(e->device));
    CUDA_CHECK(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    GameP& P = e->P;
    P.kind = gd.kind; P.m = gd.m; P.n = gd.n; P.k = gd.k; P.cells = gd.m * gd.n;
    P.A = gd.kind == AZ_GAME_C4 ? gd.n : P.cells;
    P.komi = gd.komi; P.max_moves = gd.max_moves; P.maxDepth = m.m * m.n; P.puct = m.puct; P.sims = m.sims;
    P.dont_prefer_pass = m.pass_preference == 0; P.dumb_pass = m.dumb_pass != 0; P.dont_resign = m.pass_preference == 2;
    P.resign_pct = m.resign_percentage;
    P.wq_complete = (gd.kind == AZ_GAME_WQ && (desc->flags & AZ_FLAG_WQ_COMPLETE)) ? 1 : 0;
    P.random_count = m.random_count; P.random_min_visits = m.random_min_visits; P.random_temperature = m.random_temperature; P.shared_tree = (desc->flags & AZ_FLAG_SHARED_TREE) ? 1 : 0;
    P.encoder = desc->encoder; P.F = n.features; P.plane = n.features * P.cells;
    P.hist_len = desc->encoder == AZ_ENC_WQ18 ? 8 : 0;
    if (desc->encoder == AZ_ENC_WQ18 && n.features != 18) throw std::runtime_error("WQEncoder produces 18 planes");
    if (desc->encoder == AZ_ENC_TWO_PLANE && n.features != 2) throw std::runtime_error("two-plane encoder produces 2 planes");
    P.max_plies = gd.max_moves > 0 ? gd.max_moves + 2 : (gd.kind == AZ_GAME_MNK ? P.cells + 2 : 1024);
    const bool reuse = gd.kind == AZ_GAME_MNK;
    long long auto_nodes = (long long)(m.sims + 2) * (P.A + 1 + 3) * (reuse ? (P.cells + 1) : 1) + 16;  // +3: block alignment
    P.max_nodes = desc->max_nodes_per_tree > 0 ? desc->max_nodes_per_tree : (int)std::min<long long>(auto_nodes, 1LL << 30);
    P.max_nodes = (P.max_nodes + 3) & ~3;
    if (P.maxDepth < 1) throw std::runtime_error("mcts.Config M*N must be >= 1");

    EngineDev& E = e->E;
    const int G = desc->n_games;
    E.G = G; E.T = P.shared_tree ? 1 : 2; E.cellsP = (P.cells + 15) & ~15;
    const int V = desc->mcts.workers > 1 ? desc->mcts.workers : 1;
    if (V > 4096 || (long long)G * V > (1LL << 24)) throw std::runtime_error("mcts.Config workers out of range");
    E.V = V; E.GS = G * V;
    const size_t GV = (size_t)G * V;
    E.Lmax = std::max(n.action_space, P.A + 1);
    E.tree_seed = derive_seed(desc->seed, 1);
    E.board = e->dalloc<uint8_t>((size_t)G * E.cellsP);
    E.hist = e->dalloc<uint8_t>(P.hist_len ? (size_t)G * 8 * E.cellsP : 1);
    E.gi = e->dalloc<int32_t>((size_t)G * GI_COUNT);
    E.moves = e->dalloc<int16_t>((size_t)G * P.max_plies);
    E.hmoves = e->dalloc<int16_t>((size_t)G * P.max_plies);
    const size_t GT = (size_t)G * E.T;
    E.ti = e->dalloc<int32_t>(GT * TI_COUNT);
    E.pol_hash = e->dalloc<uint32_t>(GT * P.max_plies);
    E.pol_move = e->dalloc<int16_t>(GT * P.max_plies);
    const size_t NN = GT * (size_t)P.max_nodes;
    E.N = e->dalloc<uint32_t>(NN, false); E.W = e->dalloc<float>(NN, false); E.Pr = e->dalloc<float>(NN, false);
    E.meta = e->dalloc<uint32_t>(NN, false); E.first = e->dalloc<int32_t>(NN, false);
    E.wv = e->dalloc<int32_t>(GV * WV_COUNT);
    E.path = e->dalloc<int32_t>(GV * (P.maxDepth + 1));
    E.leaf_board = e->dalloc<uint8_t>(GV * E.cellsP);
    E.batch_count = e->dalloc<int32_t>(4);
    E.nn_in = e->dalloc<float>((size_t)2 * GV * P.plane);
    E.policy = e->dalloc<float>((size_t)2 * GV * E.Lmax);
    E.value = e->dalloc<float>((size_t)2 * GV);
    E.vl = V > 1 ? e->dalloc<uint8_t>(NN) : nullptr;
    e->round_workers_dev = e->dalloc<int32_t>(1);
    E.round_workers = e->round_workers_dev;
    E.ex_board = e->dalloc<float>((size_t)G * P.plane);
    E.ex_policy = e->dalloc<float>((size_t)G * (P.A + 1));
    E.ex_value = e->dalloc<float>(G);
    E.ex_valid = e->dalloc<int32_t>(G);
    E.err = e->dalloc<int32_t>(1);
    E.counters = e->dalloc<unsigned long long>(CNT_COUNT);
    E.n_active = e->dalloc<int32_t>(1);
    {  // zobrist table (wq/zobrist.go:31-41): r.Int31() per entry, injected seed
      std::vector<int32_t> zt((size_t)P.cells * 2);
      uint64_t s = gd.zobrist_seed;
      for (auto& v : zt) v = (int32_t)(splitmix64(&s) >> 33);
      int32_t* z = e->dalloc<int32_t>(zt.size());
      CUDA_CHECK(cudaMemcpy(z, zt.data(), zt.size() * 4, cudaMemcpyHostToDevice));
      E.ztable = z;
    }
    E.zt64 = nullptr; E.poshash = nullptr; E.pathhash = nullptr;
    if (P.wq_complete) {  // positional superko: 64-bit position keys from their own stream of the zobrist seed
      e->zt64.resize((size_t)P.cells * 2);
      uint64_t s = derive_seed(gd.zobrist_seed, 0x706f736974696f6eull);
      for (auto& v : e->zt64) v = splitmix64(&s);
      unsigned long long* z = e->dalloc<unsigned long long>(e->zt64.size());
      CUDA_CHECK(cudaMemcpy(z, e->zt64.data(), e->zt64.size() * 8, cudaMemcpyHostToDevice));
      E.zt64 = z;
      E.poshash = e->dalloc<unsigned long long>((size_t)G * (P.max_plies + 2));
      E.pathhash = e->dalloc<unsigned long long>(GV * (P.maxDepth + 2));
    }
    for (int a = 0; a < 2; a++) { E.inf[a].kind = -1; E.inf[a].L = n.action_space; E.inf[a].dummy_value = 0; E.inf[a].table = nullptr; E.inf[a].table_values = nullptr; E.inf[a].table_rows = 0; }
    e->coins_dev = e->dalloc<int>(G);
    if (const char* ng = getenv("AZ_NO_GRAPH")) e->graphs_enabled = !(ng[0] == '1');
    e->coin_state = derive_seed(desc->seed, 0);
    mcts_set_smem_limits(P, E.cellsP);
    heads_tiled_configure();

    NetDims nd;
    nd.K = n.k; nd.SharedLayers = n.shared_layers; nd.FC = n.fc; nd.B = n.batch_size; nd.W = n.width; nd.H = n.height;
    nd.F = n.features; nd.A1 = n.action_space;
    e->L = build_layout(nd);
    for (int a = 0; a < 2; a++) {
      e->net_params[a] = e->dalloc<float>(e->L.total + 4);  // +4: the fused collective moves float4s
      e->snap[a] = make_snapshot_layout(e->L);
      e->snap[a].d = e->dalloc<float>(e->snap[a].total);
    }
    fp32_scratch_alloc(e->fp32, nd, E.GS);
    e->use_tc = !(desc->flags & AZ_FLAG_FP32_TOWER) && tc_tower_supported(nd);
    if (e->use_tc)
      for (int a = 0; a < 2; a++) tc_tower_alloc(e->tc[a], nd, E.GS, desc->act_scale_log2 ? desc->act_scale_log2 : -2);

    CUDA_CHECK(cudaMallocHost(&e->h_ex_board, (size_t)G * P.plane * 4));
    CUDA_CHECK(cudaMallocHost(&e->h_ex_policy, (size_t)G * (P.A + 1) * 4));
    CUDA_CHECK(cudaMallocHost(&e->h_ex_value, (size_t)G * 4));
    CUDA_CHECK(cudaMallocHost(&e->h_ex_valid, (size_t)G * 4));
    CUDA_CHECK(cudaMallocHost(&e->h_small, 64));
    CUDA_CHECK(cudaDeviceSynchronize());
  } catch (const CudaError& ce2) {
    g_create_error = ce2.msg; az_engine_destroy(e.release()); return AZ_ERR_CUDA;
  } catch (const std::exception& ex) {
    g_create_error = ex.what(); az_engine_destroy(e.release()); return AZ_ERR_INVALID;
  }
  *out = e.release();
  return AZ_OK;
}

// ---- nets -------------------------------------------------------------------------------------
int az_net_param_count(const az_engine* e, int32_t* n_tensors, uint64_t* n_floats) {
  if (n_tensors) *n_tensors = (int32_t)e->L.desc.size();
  if (n_floats) *n_floats = e->L.total;
  return AZ_OK;
}
int az_net_param_desc(const az_engine* e, int32_t i, char name[96], int32_t shape[4], int32_t* rank, uint64_t* offset,
                      uint64_t* size) {
  if (i < 0 || i >= (int)e->L.desc.size()) return AZ_ERR_INVALID;
  const ParamDescH& d = e->L.desc[i];
  if (name) snprintf(name, 96, "%s", d.name.c_str());
  if (shape) for (int k = 0; k < 4; k++) shape[k] = d.shape[k];
  if (rank) *rank = d.rank;
  if (offset) *offset = d.offset;
  if (size) *size = d.size;
  return AZ_OK;
}
int az_net_init(az_engine* e, int32_t net, uint64_t seed) {
  if (net < 0 || net > 1) return AZ_ERR_INVALID;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  std::vector<float> h;
  init_params_host(e->L, seed, &h);
  CUDA_CHECK(cudaMemcpy(e->net_params[net], h.data(), h.size() * 4, cudaMemcpyHostToDevice));
  GUARD_END(e)
  return AZ_OK;
}
int az_net_get_params(az_engine* e, int32_t net, float* out, uint64_t n) {
  if (net < 0 || net > 1 || n != e->L.total) return AZ_ERR_INVALID;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  CUDA_CHECK(cudaMemcpy(out, e->net_params[net], n * 4, cudaMemcpyDeviceToHost));
  GUARD_END(e)
  return AZ_OK;
}
int az_net_set_params(az_engine* e, int32_t net, const float* in, uint64_t n) {
  if (net < 0 || net > 1 || n != e->L.total) return AZ_ERR_INVALID;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  CUDA_CHECK(cudaMemcpy(e->net_params[net], in, n * 4, cudaMemcpyHostToDevice));
  GUARD_END(e)
  return AZ_OK;
}
int az_net_copy(az_engine* e, int32_t dst, int32_t src) {
  if (dst < 0 || dst > 1 || src < 0 || src > 1) return AZ_ERR_INVALID;
  if (dst == src) return AZ_OK;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  CUDA_CHECK(cudaMemcpyAsync(e->net_params[dst], e->net_params[src], e->L.total * 4, cudaMemcpyDeviceToDevice, e->stream));
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  GUARD_END(e)
  return AZ_OK;
}

// ---- agents -----------------------------------------------------------------------------------
int az_agent_set_inferer(az_engine* e, int32_t agent, int32_t kind, int32_t dummy_player) {
  if (agent < 0 || agent > 1) return AZ_ERR_INVALID;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  InfererDev& I = e->E.inf[agent];
  if (kind == AZ_INF_DUAL) {
    snapshot_gather(e->L, e->net_params[agent], e->snap[agent], e->stream);
    if (e->use_tc) tc_tower_prepare(e->tc[agent], e->snap[agent], e->stream);
    CUDA_CHECK(cudaStreamSynchronize(e->stream));
    e->snap_valid[agent] = true;
    I.kind = INF_DUAL; I.L = e->d.nn.action_space;
  } else if (kind == AZ_INF_DUMMY) {
    I.kind = INF_DUMMY; I.L = e->P.A;  // dummy.go: outputSize = g.ActionSpace()
    I.dummy_value = dummy_player == 1 ? 1.0f : (dummy_player == 2 ? -1.0f : 0.0f);
  } else if (kind == AZ_INF_TABLE) {
    I.kind = INF_TABLE;
  } else return AZ_ERR_INVALID;
  e->inf_kind[agent] = kind;
  e->cfg_version++;
  GUARD_END(e)
  return AZ_OK;
}
int az_agent_set_table(az_engine* e, int32_t agent, int32_t n_rows, int32_t row_len, const float* policy_rows,
                       const float* values) {
  if (agent < 0 || agent > 1 || n_rows < 1 || row_len < 1) return AZ_ERR_INVALID;
  if (row_len > e->E.Lmax || row_len < e->P.A) { e->err = "table row length must be in [ActionSpace, ActionSpace+1]"; return AZ_ERR_INVALID; }
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  // a table replaces the agent's previous one: free that first (dalloc keeps every allocation until destroy)
  for (float* old : {e->table_dev[agent], e->table_val_dev[agent]})
    if (old) { auto it = std::find(e->allocs.begin(), e->allocs.end(), (void*)old); if (it != e->allocs.end()) e->allocs.erase(it); CUDA_CHECK(cudaStreamSynchronize(e->stream)); cudaFree(old); }
  float* t = e->dalloc<float>((size_t)n_rows * row_len);
  float* v = e->dalloc<float>(n_rows);
  e->table_dev[agent] = t; e->table_val_dev[agent] = v;
  CUDA_CHECK(cudaMemcpy(t, policy_rows, (size_t)n_rows * row_len * 4, cudaMemcpyHostToDevice));
  CUDA_CHECK(cudaMemcpy(v, values, (size_t)n_rows * 4, cudaMemcpyHostToDevice));
  InfererDev& I = e->E.inf[agent];
  I.kind = INF_TABLE; I.L = row_len; I.table = t; I.table_values = v; I.table_rows = n_rows;
  e->inf_kind[agent] = AZ_INF_TABLE;
  e->cfg_version++;
  GUARD_END(e)
  return AZ_OK;
}

// forward of one agent's pending batch (count on device); returns the fp32 tower's output buffer (nullptr on the
// tensor-core tower, whose output stays in its own fp16 hi/lo layout)
static const float* run_forward(az_engine* e, int agent, cudaStream_t st = nullptr) {
  if (!st) st = e->stream;
  const EngineDev& E = e->E;
  if (E.inf[agent].kind != INF_DUAL) return nullptr;
  const float* in = E.nn_in + (size_t)agent * E.GS * e->P.plane;
  float* pol = E.policy + (size_t)agent * E.GS * E.Lmax;
  float* val = E.value + (size_t)agent * E.GS;
  const int* cnt = E.batch_count + agent;
  if (e->use_tc) { tc_tower_forward(e->tc[agent], e->L, e->snap[agent], e->fp32, in, cnt, E.GS, pol, E.Lmax, val, E.err, st, &e->launches); return nullptr; }
  return forward_fp32(e->L, e->snap[agent], e->fp32, in, cnt, E.GS, pol, E.Lmax, val, st, &e->launches);
}

int az_infer(az_engine* e, int32_t agent, const float* planes, int32_t n, float* policy, float* value) {
  if (agent < 0 || agent > 1 || n < 0) return AZ_ERR_INVALID;
  if (e->E.inf[agent].kind != INF_DUAL || !e->snap_valid[agent]) { e->err = "agent has no dual inferer (call az_agent_set_inferer(AZ_INF_DUAL))"; return AZ_ERR_STATE; }
  if (e->in_play) { e->err = "az_infer during a running arena"; return AZ_ERR_STATE; }
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  const EngineDev& E = e->E;
  const int A1 = e->d.nn.action_space;
  for (int done = 0; done < n; done += E.GS) {
    int chunk = std::min(E.GS, n - done);
    CUDA_CHECK(cudaMemcpyAsync(E.nn_in + (size_t)agent * E.GS * e->P.plane, planes + (size_t)done * e->P.plane,
                               (size_t)chunk * e->P.plane * 4, cudaMemcpyHostToDevice, e->stream));
    CUDA_CHECK(cudaMemcpyAsync(E.batch_count + agent, &chunk, 4, cudaMemcpyHostToDevice, e->stream));
    run_forward(e, agent);
    CUDA_CHECK(cudaMemcpy2DAsync(policy + (size_t)done * A1, (size_t)A1 * 4, E.policy + (size_t)agent * E.GS * E.Lmax,
                                 (size_t)E.Lmax * 4, (size_t)A1 * 4, chunk, cudaMemcpyDeviceToHost, e->stream));
    CUDA_CHECK(cudaMemcpyAsync(value + done, E.value + (size_t)agent * E.GS, (size_t)chunk * 4, cudaMemcpyDeviceToHost, e->stream));
    CUDA_CHECK(cudaStreamSynchronize(e->stream));
  }
  int bits = 0;
  CUDA_CHECK(cudaMemcpy(&bits, E.err, 4, cudaMemcpyDeviceToHost));
  if (bits) { CUDA_CHECK(cudaMemsetAsync(E.err, 0, 4, e->stream)); return device_error_to_rc(e, bits); }
  GUARD_END(e)
  return AZ_OK;
}
int az_infer_tower(az_engine* e, int32_t agent, const float* planes, int32_t n, float* tower_out) {
  if (agent < 0 || agent > 1 || n < 0) return AZ_ERR_INVALID;
  if (e->E.inf[agent].kind != INF_DUAL || !e->snap_valid[agent]) { e->err = "agent has no dual inferer (call az_agent_set_inferer(AZ_INF_DUAL))"; return AZ_ERR_STATE; }
  if (e->in_play) { e->err = "az_infer_tower during a running arena"; return AZ_ERR_STATE; }
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  const EngineDev& E = e->E;
  const size_t per = (size_t)e->L.d.K * e->L.d.HW();
  for (int done = 0; done < n; done += E.GS) {
    int chunk = std::min(E.GS, n - done);
    CUDA_CHECK(cudaMemcpyAsync(E.nn_in + (size_t)agent * E.GS * e->P.plane, planes + (size_t)done * e->P.plane,
                               (size_t)chunk * e->P.plane * 4, cudaMemcpyHostToDevice, e->stream));
    CUDA_CHECK(cudaMemcpyAsync(E.batch_count + agent, &chunk, 4, cudaMemcpyHostToDevice, e->stream));
    const float* tower = run_forward(e, agent);
    if (e->use_tc) {  // the fp32 tower's scratch is idle on this engine: unpack the hi/lo output into it
      tc_tower_output(e->tc[agent], E.batch_count + agent, E.GS, e->fp32.a, e->stream);
      tower = e->fp32.a;
    }
    CUDA_CHECK(cudaMemcpyAsync(tower_out + (size_t)done * per, tower, (size_t)chunk * per * 4, cudaMemcpyDeviceToHost, e->stream));
    CUDA_CHECK(cudaStreamSynchronize(e->stream));
  }
  int bits = 0;
  CUDA_CHECK(cudaMemcpy(&bits, E.err, 4, cudaMemcpyDeviceToHost));
  if (bits) { CUDA_CHECK(cudaMemsetAsync(E.err, 0, 4, e->stream)); return device_error_to_rc(e, bits); }
  GUARD_END(e)
  return AZ_OK;
}
int az_agent_stats(const az_engine* e, int32_t agent, float* wins, float* loss, float* draw) {
  if (agent < 0 || agent > 1) return AZ_ERR_INVALID;
  *wins = e->wins[agent]; *loss = e->loss[agent]; *draw = e->draw[agent];
  return AZ_OK;
}
int az_agent_reset_stats(az_engine* e, int32_t agent) {
  if (agent < 0 || agent > 1) return AZ_ERR_INVALID;
  e->wins[agent] = e->loss[agent] = e->draw[agent] = 0;
  return AZ_OK;
}

// ---- arena ------------------------------------------------------------------------------------
static int sync_small(az_engine* e, int* n_active) {
  const EngineDev& E = e->E;
  CUDA_CHECK(cudaMemcpyAsync(e->h_small, E.n_active, 4, cudaMemcpyDeviceToHost, e->stream));
  CUDA_CHECK(cudaMemcpyAsync(e->h_small + 1, E.err, 4, cudaMemcpyDeviceToHost, e->stream));
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  if (n_active) *n_active = e->h_small[0];
  int bits = e->h_small[1];
  if (bits) { CUDA_CHECK(cudaMemsetAsync(E.err, 0, 4, e->stream)); return device_error_to_rc(e, bits); }
  return AZ_OK;
}

int az_arena_begin(az_engine* e, int32_t n_games, int32_t record) {
  if (n_games < 1 || n_games > e->E.G) { e->err = "n_games out of range"; return AZ_ERR_INVALID; }
  const bool shared = e->P.shared_tree;
  if (e->E.inf[0].kind < 0 || (!shared && e->E.inf[1].kind < 0)) { e->err = "agents have no inferer"; return AZ_ERR_STATE; }
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  std::vector<int> coins(n_games);
  for (int g = 0; g < n_games; g++) coins[g] = (int)(splitmix64(&e->coin_state) % 2);  // arena.go:81 a.r.Intn(2)
  CUDA_CHECK(cudaMemcpyAsync(e->coins_dev, coins.data(), (size_t)n_games * 4, cudaMemcpyHostToDevice, e->stream));
  launch_arena_begin(e->P, e->E, n_games, e->coins_dev, e->games_started, e->stream); e->launches++;
  e->games_started += (uint64_t)n_games;
  launch_assign_slots(e->P, e->E, n_games, e->stream); e->launches++;
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  e->in_play = true; e->record = record != 0; e->n_play = n_games;
  e->ext_prev[0].valid = e->ext_prev[1].valid = false;  // the arena owns slot 0 now
  e->ex_by_game.assign(n_games, {});
  e->records.clear();
  GUARD_END(e)
  return AZ_OK;
}

static void eval_pending(az_engine* e) {
  launch_infer_simple(e->P, e->E, e->n_play, e->stream); e->launches++;
  run_forward(e, 0);
  if (!e->P.shared_tree) run_forward(e, 1);
  launch_expand_backup(e->P, e->E, e->n_play, e->stream); e->launches++;
}

int az_search_begin(az_engine* e) {
  if (!e->in_play) return AZ_ERR_STATE;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  launch_assign_slots(e->P, e->E, e->n_play, e->stream); e->launches++;
  launch_search_begin(e->P, e->E, e->n_play, e->stream); e->launches++;
  launch_encode_roots(e->P, e->E, e->n_play, e->stream); e->launches++;
  eval_pending(e);
  GUARD_END_PLAY(e)
  return AZ_OK;
}
// n pipeline iterations = ceil(n / workers) rounds; the device reads how many workers the round starts
static void set_round_workers(az_engine* e, int w) {
  if (e->E.V == 1 || e->round_workers_host == w) return;
  e->round_workers_host = w;
  CUDA_CHECK(cudaMemcpyAsync(e->round_workers_dev, &e->round_workers_host, 4, cudaMemcpyHostToDevice, e->stream));
}
static void run_wave(az_engine* e) {
  launch_select(e->P, e->E, e->n_play, e->stream); e->launches++;
  eval_pending(e);
}
int az_search_run(az_engine* e, int32_t n) {
  if (!e->in_play) return AZ_ERR_STATE;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  if (e->graphs_enabled && !e->profiling && n >= 1) {
    if (!e->wave_graph || e->wave_graph_n != e->n_play || e->wave_graph_version != e->cfg_version) {
      if (e->wave_graph) { cudaGraphExecDestroy(e->wave_graph); e->wave_graph = nullptr; }
      const unsigned long long l0 = e->launches;
      cudaGraph_t g = nullptr;
      CUDA_CHECK(cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal));
      try { run_wave(e); } catch (...) { cudaStreamEndCapture(e->stream, &g); if (g) cudaGraphDestroy(g); throw; }
      CUDA_CHECK(cudaStreamEndCapture(e->stream, &g));
      CUDA_CHECK(cudaGraphInstantiate(&e->wave_graph, g, 0));
      cudaGraphDestroy(g);
      e->wave_graph_launches = e->launches - l0;
      e->launches = l0;
      e->wave_graph_n = e->n_play; e->wave_graph_version = e->cfg_version;
    }
    for (int left = n; left > 0; left -= e->E.V) {
      set_round_workers(e, std::min(left, e->E.V));
      CUDA_CHECK(cudaGraphLaunch(e->wave_graph, e->stream)); e->launches += e->wave_graph_launches;
    }
  } else {
    for (int left = n; left > 0; left -= e->E.V) { set_round_workers(e, std::min(left, e->E.V)); run_wave(e); }
  }
  GUARD_END_PLAY(e)
  return AZ_OK;
}
int az_search_end(az_engine* e) {
  if (!e->in_play) return AZ_ERR_STATE;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  const EngineDev& E = e->E;
  const GameP& P = e->P;
  launch_search_end(P, E, e->n_play, e->record ? 1 : 0, e->stream); e->launches++;
  launch_assign_slots(P, E, e->n_play, e->stream); e->launches++;  // refreshes n_active
  const int n = e->n_play;
  if (e->record) {
    CUDA_CHECK(cudaMemcpyAsync(e->h_ex_valid, E.ex_valid, (size_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
    CUDA_CHECK(cudaMemcpyAsync(e->h_ex_value, E.ex_value, (size_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
    CUDA_CHECK(cudaMemcpyAsync(e->h_ex_policy, E.ex_policy, (size_t)n * (P.A + 1) * 4, cudaMemcpyDeviceToHost, e->stream));
    CUDA_CHECK(cudaMemcpyAsync(e->h_ex_board, E.ex_board, (size_t)n * P.plane * 4, cudaMemcpyDeviceToHost, e->stream));
  }
  int rc = sync_small(e, nullptr);
  if (rc) { PLAY_ABORT(e); return rc; }
  if (e->record) {
    for (int g = 0; g < n; g++) {
      if (!e->h_ex_valid[g]) continue;
      HostExample ex;
      ex.board.assign(e->h_ex_board + (size_t)g * P.plane, e->h_ex_board + (size_t)(g + 1) * P.plane);
      ex.policy.assign(e->h_ex_policy + (size_t)g * (P.A + 1), e->h_ex_policy + (size_t)(g + 1) * (P.A + 1));
      ex.value = e->h_ex_value[g];
      e->ex_by_game[g].push_back(std::move(ex));
    }
  }
  GUARD_END_PLAY(e)
  return AZ_OK;
}
int az_arena_step(az_engine* e, int32_t* n_active) {
  int rc;
  if ((rc = az_search_begin(e))) return rc;
  if ((rc = az_search_run(e, e->P.sims))) return rc;
  if ((rc = az_search_end(e))) return rc;
  if (n_active) *n_active = e->h_small[0];
  return AZ_OK;
}

static void read_games(az_engine* e, std::vector<int32_t>* gi, std::vector<int16_t>* moves) {
  const EngineDev& E = e->E;
  gi->resize((size_t)e->n_play * GI_COUNT);
  moves->resize((size_t)e->n_play * e->P.max_plies);
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  CUDA_CHECK(cudaMemcpy(gi->data(), E.gi, gi->size() * 4, cudaMemcpyDeviceToHost));
  CUDA_CHECK(cudaMemcpy(moves->data(), E.moves, moves->size() * 2, cudaMemcpyDeviceToHost));
}

int az_arena_finish(az_engine* e) {
  if (!e->in_play) return AZ_ERR_STATE;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  std::vector<int32_t> gi; std::vector<int16_t> moves;
  read_games(e, &gi, &moves);
  e->records.clear();
  for (int g = 0; g < e->n_play; g++) {
    const int32_t* G = gi.data() + (size_t)g * GI_COUNT;
    HostRecord r;
    r.winner = G[GI_WINNER]; r.a_player = G[GI_A_PLAYER];
    for (int i = 0; i < G[GI_N_MOVES]; i++) r.moves.push_back(moves[(size_t)g * e->P.max_plies + i]);
    // arena.go:146-155 labels ; 156-169 win/loss/draw
    for (HostExample& ex : e->ex_by_game[g]) {
      if (r.winner == AZ_NONE) ex.value = 0;
      else if (ex.value == (float)r.winner) ex.value = 1;
      else ex.value = -1;
      e->examples.push_back(std::move(ex));
    }
    r.n_examples = (int)e->ex_by_game[g].size();
    int b_player = r.a_player == AZ_BLACK ? AZ_WHITE : AZ_BLACK;
    if (r.winner == AZ_NONE) { e->draw[0]++; e->draw[1]++; }
    else if (r.winner == r.a_player) { e->wins[0]++; e->loss[1]++; }
    else if (r.winner == b_player) { e->wins[1]++; e->loss[0]++; }
    e->records.push_back(std::move(r));
  }
  e->ex_by_game.clear();
  e->in_play = false;
  GUARD_END_PLAY(e)
  return AZ_OK;
}
int az_arena_play(az_engine* e, int32_t n_games, int32_t record) {
  int done = 0;
  std::vector<HostRecord> all;
  while (done < n_games) {
    int chunk = std::min(n_games - done, e->E.G);
    int rc;
    if ((rc = az_arena_begin(e, chunk, record))) return rc;
    int na = chunk;
    // games that are already over (cannot happen on an empty board) would show up as n_active == 0
    while (na > 0) if ((rc = az_arena_step(e, &na))) return rc;
    if ((rc = az_arena_finish(e))) return rc;
    for (auto& r : e->records) all.push_back(r);
    done += chunk;
  }
  e->records = all;
  return AZ_OK;
}

int az_search(az_engine* e, int32_t agent, const az_state* st, int32_t player, int32_t* best, float* child_visits) {
  if (agent < 0 || agent > 1 || !st || !st->board || st->n_hist < 0 || (st->n_hist > 0 && !st->hist)) return AZ_ERR_INVALID;
  if (st->n_hist > (e->P.wq_complete ? e->P.max_plies : 8)) return AZ_ERR_INVALID;  // complete rules: superko reads them all
  if (e->in_play) { e->err = "az_search during a running arena"; return AZ_ERR_STATE; }
  if (e->E.inf[agent].kind < 0) { e->err = "agent has no inferer"; return AZ_ERR_STATE; }
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  const GameP& P = e->P;
  const EngineDev& E = e->E;
  // ---- newRootState (search.go:424-469) on the host: may the agent's tree be re-rooted on this position?
  const int t_idx = P.shared_tree ? 0 : agent;
  az_engine::ExtPrev& prev = e->ext_prev[t_idx];
  std::vector<uint8_t> b(E.cellsP, 0);
  for (int i = 0; i < P.cells; i++) b[i] = (uint8_t)st->board[i];
  int depth = st->move_number - prev.move_number;
  bool reuse = P.kind == KIND_MNK && prev.valid && depth >= 0 && (depth == 0 || (st->moves && st->n_moves >= depth)) &&
               st->move_number < P.max_plies;
  if (reuse) {  // tmp.UndoLastMove() x depth, then tmp.Eq(prev): mnk's Undo clears the cell of each undone move (mnk.go:184-189)
    std::vector<uint8_t> tmp = b;
    for (int i = 0; i < depth && reuse; i++) {
      const int mv = st->moves[2 * (st->n_moves - 1 - i) + 1];
      if (mv < 0 || mv >= P.cells) reuse = false; else tmp[mv] = 0;
    }
    if (reuse) reuse = memcmp(tmp.data(), prev.board.data(), P.cells) == 0;
  }
  if (!reuse) {
    // fresh tree for this agent (the other agent's tree in slot 0 is untouched): empty pool, no root, RNG stream t of the
    // engine's tree seed (what k_arena_begin gives tree t of the first game)
    const uint64_t ts = derive_seed(E.tree_seed, (uint64_t)t_idx);
    int32_t tiv[TI_COUNT] = {0};
    tiv[TI_ROOT] = -1; tiv[TI_RNG_LO] = (int32_t)(uint32_t)(ts & 0xffffffffu); tiv[TI_RNG_HI] = (int32_t)(uint32_t)(ts >> 32);
    CUDA_CHECK(cudaMemcpyAsync(E.ti + (size_t)t_idx * TI_COUNT, tiv, sizeof tiv, cudaMemcpyHostToDevice, e->stream));
    CUDA_CHECK(cudaMemsetAsync(E.wv, 0, (size_t)E.V * WV_COUNT * 4, e->stream));
    CUDA_CHECK(cudaStreamSynchronize(e->stream));  // tiv is a stack buffer
    prev.valid = false;
  } else {
    // keep the tree: reset only the per-search worker records of slot 0 and hand the replay (Fwd + findChild per move)
    // to k_search_begin through the slot's move history
    CUDA_CHECK(cudaMemsetAsync(E.wv, 0, (size_t)E.V * WV_COUNT * 4, e->stream));
    std::vector<int16_t> hm(depth > 0 ? depth : 1);
    for (int i = 0; i < depth; i++) hm[i] = (int16_t)st->moves[2 * (st->n_moves - depth + i) + 1];
    if (depth > 0) CUDA_CHECK(cudaMemcpyAsync(E.hmoves + prev.move_number, hm.data(), (size_t)depth * 2, cudaMemcpyHostToDevice, e->stream));
    int32_t pv[3] = {1, prev.move_number, 0};  // TI_PREV_VALID, TI_PREV_MN, TI_NPOL (cachedPolicies only feed Arena examples)
    static_assert(TI_PREV_MN == TI_PREV_VALID + 1 && TI_NPOL == TI_PREV_VALID + 2, "tree-info layout");
    CUDA_CHECK(cudaMemcpyAsync(E.ti + (size_t)t_idx * TI_COUNT + TI_PREV_VALID, pv, 12, cudaMemcpyHostToDevice, e->stream));
    CUDA_CHECK(cudaStreamSynchronize(e->stream));  // hm / pv are stack buffers
  }
  std::vector<uint8_t> ring(P.hist_len ? (size_t)8 * E.cellsP : 1, 0);
  if (P.hist_len)
    for (int i = std::max(0, st->n_hist - 8); i < st->n_hist; i++) {  // the encoder looks back 8 boards
      int h = st->move_number - st->n_hist + i;  // Historical(h) = board before move h
      if (h < 0) continue;
      for (int c = 0; c < P.cells; c++) ring[(size_t)(h & 7) * E.cellsP + c] = (uint8_t)st->hist[(size_t)i * P.cells + c];
    }
  int32_t gi[GI_COUNT] = {0};
  const int opp_player = player == AZ_BLACK ? AZ_WHITE : AZ_BLACK;
  gi[GI_TO_MOVE] = st->to_move; gi[GI_MOVE_NUMBER] = st->move_number;
  gi[GI_PASSES] = P.kind == KIND_MNK ? -1 : (P.kind == KIND_WQ ? st->passes : 0);
  gi[GI_C4_PASS] = P.kind == KIND_C4 ? st->passes : 0;
  gi[GI_ACTIVE] = 1; gi[GI_CUR_AGENT] = P.shared_tree ? 0 : agent; gi[GI_LAST_MOVE] = st->last_move;
  gi[GI_KO] = P.wq_complete ? st->ko : -1;
  gi[GI_A_PLAYER] = (P.shared_tree || agent == 0) ? player : opp_player;
  if (P.kind == KIND_WQ) {  // clean Zobrist hash of the position (wq/zobrist.go:44-56)
    std::vector<int32_t> zt((size_t)P.cells * 2);
    CUDA_CHECK(cudaMemcpy(zt.data(), E.ztable, zt.size() * 4, cudaMemcpyDeviceToHost));
    int32_t h = 0;
    for (int i = 0; i < P.cells; i++) if (st->board[i]) h ^= zt[i * 2 + (st->board[i] == AZ_BLACK ? 0 : 1)];
    gi[GI_ZHASH] = h;
  }
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  CUDA_CHECK(cudaMemcpy(E.board, b.data(), b.size(), cudaMemcpyHostToDevice));
  if (P.hist_len) CUDA_CHECK(cudaMemcpy(E.hist, ring.data(), ring.size(), cudaMemcpyHostToDevice));
  if (E.poshash) {  // positional superko sees the boards the caller supplies (the earlier positions of the game), then the current one
    std::vector<unsigned long long> ph;
    auto hash_of = [&](const int32_t* bd) {
      unsigned long long h = 0;
      for (int c = 0; c < P.cells; c++) if (bd[c]) h ^= e->zt64[(size_t)c * 2 + (bd[c] == AZ_BLACK ? 0 : 1)];
      return h;
    };
    for (int i = 0; i < st->n_hist; i++)
      if (st->move_number - st->n_hist + i >= 0) ph.push_back(hash_of(st->hist + (size_t)i * P.cells));
    while ((int)ph.size() > P.max_plies) ph.erase(ph.begin());  // the row holds max_plies + 2 entries
    gi[GI_N_POS] = (int32_t)ph.size();
    ph.push_back(hash_of(st->board));
    CUDA_CHECK(cudaMemcpy(E.poshash, ph.data(), ph.size() * 8, cudaMemcpyHostToDevice));
  }
  CUDA_CHECK(cudaMemcpy(E.gi, gi, sizeof gi, cudaMemcpyHostToDevice));
  e->in_play = true; e->record = false; e->n_play = 1;
  e->ex_by_game.assign(1, {});
  int rc = az_search_begin(e);
  if (!rc) rc = az_search_run(e, P.sims);
  // visit counts of the root's children, before the epilogue permutes/applies anything that matters to us
  if (!rc && child_visits) {
    const int t = P.shared_tree ? 0 : agent;
    CUDA_CHECK(cudaStreamSynchronize(e->stream));
    int32_t ti[TI_COUNT];
    CUDA_CHECK(cudaMemcpy(ti, E.ti + (size_t)t * TI_COUNT, sizeof ti, cudaMemcpyDeviceToHost));
    for (int i = 0; i <= P.A; i++) child_visits[i] = 0;
    if (ti[TI_ROOT] >= 0) {
      const size_t tb = (size_t)t * P.max_nodes;
      uint32_t rmeta; int32_t rfirst;
      CUDA_CHECK(cudaMemcpy(&rmeta, E.meta + tb + ti[TI_ROOT], 4, cudaMemcpyDeviceToHost));
      CUDA_CHECK(cudaMemcpy(&rfirst, E.first + tb + ti[TI_ROOT], 4, cudaMemcpyDeviceToHost));
      const int nc = META_NCHILD(rmeta);
      std::vector<uint32_t> cm(nc), cn(nc);
      if (nc) {
        CUDA_CHECK(cudaMemcpy(cm.data(), E.meta + tb + rfirst, (size_t)nc * 4, cudaMemcpyDeviceToHost));
        CUDA_CHECK(cudaMemcpy(cn.data(), E.N + tb + rfirst, (size_t)nc * 4, cudaMemcpyDeviceToHost));
      }
      for (int j = 0; j < nc; j++) {
        int mv = META_MOVE(cm[j]);
        if (mv == AZ_PASS) child_visits[P.A] = (float)cn[j];
        else if (mv >= 0 && mv < P.A) child_visits[mv] = (float)cn[j];
      }
    }
  }
  if (!rc) rc = az_search_end(e);
  if (!rc && best) {
    int16_t mv;
    CUDA_CHECK(cudaMemcpy(&mv, E.moves, 2, cudaMemcpyDeviceToHost));
    *best = mv;
  }
  e->in_play = false;
  e->ex_by_game.clear();
  if (rc) { prev.valid = false; return rc; }
  // t.prev = t.current.Clone() (search.go:152): the position this tree was searched on
  prev.valid = true; prev.move_number = st->move_number; prev.board.assign(b.begin(), b.begin() + P.cells);
  GUARD_END_PLAY(e)
  return AZ_OK;
}

int az_agent_reset_tree(az_engine* e, int32_t agent) {  // MCTS.Reset (tree.go:249-276) for the external-search tree
  if (agent < 0 || agent > 1) return AZ_ERR_INVALID;
  if (e->in_play) { e->err = "az_agent_reset_tree during a running arena"; return AZ_ERR_STATE; }
  e->ext_prev[e->P.shared_tree ? 0 : agent].valid = false;
  return AZ_OK;
}

int az_game_record(const az_engine* ce, int32_t game, int32_t* moves, int32_t cap, int32_t* n_moves, int32_t* winner,
                   int32_t* a_player, int32_t* n_examples) {
  az_engine* e = const_cast<az_engine*>(ce);
  GUARD_BEGIN
  if (!e->in_play) {
    if (game < 0 || game >= (int)e->records.size()) return AZ_ERR_INVALID;
    const HostRecord& r = e->records[game];
    if (n_moves) *n_moves = (int)r.moves.size();
    if (moves) for (int i = 0; i < (int)r.moves.size() && i < cap; i++) moves[i] = r.moves[i];
    if (winner) *winner = r.winner;
    if (a_player) *a_player = r.a_player;
    if (n_examples) *n_examples = r.n_examples;
    return AZ_OK;
  }
  if (game < 0 || game >= e->n_play) return AZ_ERR_INVALID;
  CUDA_CHECK(cudaSetDevice(e->device));
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  int32_t G[GI_COUNT];
  CUDA_CHECK(cudaMemcpy(G, e->E.gi + (size_t)game * GI_COUNT, sizeof G, cudaMemcpyDeviceToHost));
  std::vector<int16_t> mv(e->P.max_plies);
  CUDA_CHECK(cudaMemcpy(mv.data(), e->E.moves + (size_t)game * e->P.max_plies, mv.size() * 2, cudaMemcpyDeviceToHost));
  if (n_moves) *n_moves = G[GI_N_MOVES];
  if (moves) for (int i = 0; i < G[GI_N_MOVES] && i < cap; i++) moves[i] = mv[i];
  if (winner) *winner = G[GI_WINNER];
  if (a_player) *a_player = G[GI_A_PLAYER];
  if (n_examples) *n_examples = (int)e->ex_by_game[game].size();
  GUARD_END(e)
  return AZ_OK;
}
int az_game_state(const az_engine* ce, int32_t game, int32_t* board, int32_t cap, int32_t* to_move, int32_t* move_number,
                  int32_t* passes, int32_t* ended, int32_t* winner) {
  az_engine* e = const_cast<az_engine*>(ce);
  if (game < 0 || game >= e->E.G) return AZ_ERR_INVALID;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  int32_t G[GI_COUNT];
  CUDA_CHECK(cudaMemcpy(G, e->E.gi + (size_t)game * GI_COUNT, sizeof G, cudaMemcpyDeviceToHost));
  std::vector<uint8_t> b(e->E.cellsP);
  CUDA_CHECK(cudaMemcpy(b.data(), e->E.board + (size_t)game * e->E.cellsP, b.size(), cudaMemcpyDeviceToHost));
  if (board) for (int i = 0; i < e->P.cells && i < cap; i++) board[i] = b[i];
  if (to_move) *to_move = G[GI_TO_MOVE];
  // MoveNumber(): mnk/wq len(history); c4 the constant moveCount+1 = 1 (c4/game.go:51)
  if (move_number) *move_number = e->P.kind == KIND_C4 ? 1 : G[GI_MOVE_NUMBER];
  if (passes) *passes = G[GI_PASSES];
  // Ended(): what Arena.Play's loop condition last saw
  if (ended) *ended = (!G[GI_ACTIVE] && G[GI_ARENA_PASS] < 2 && !(e->P.max_moves > 0 && G[GI_N_MOVES] >= e->P.max_moves)) ? 1 : 0;
  if (ended && e->P.wq_complete && !G[GI_ACTIVE] && G[GI_ARENA_PASS] >= 2) *ended = 1;  // complete rules: two passes are scored
  if (winner) *winner = G[GI_WINNER];
  GUARD_END(e)
  return AZ_OK;
}
int az_examples_count(const az_engine* e, int64_t* n) { *n = (int64_t)e->examples.size(); return AZ_OK; }
int az_examples_read(const az_engine* e, int64_t start, int64_t n, float* boards, float* policies, float* values) {
  if (start < 0 || start + n > (int64_t)e->examples.size()) return AZ_ERR_INVALID;
  for (int64_t i = 0; i < n; i++) {
    const HostExample& ex = e->examples[start + i];
    if (boards) memcpy(boards + i * ex.board.size(), ex.board.data(), ex.board.size() * 4);
    if (policies) memcpy(policies + i * ex.policy.size(), ex.policy.data(), ex.policy.size() * 4);
    if (values) values[i] = ex.value;
  }
  return AZ_OK;
}
int az_examples_clear(az_engine* e) { e->examples.clear(); return AZ_OK; }

int az_tree_dump(const az_engine* ce, int32_t game, int32_t tree, int32_t* rows, int32_t cap_rows, int32_t* n_rows) {
  az_engine* e = const_cast<az_engine*>(ce);
  const EngineDev& E = e->E;
  if (game < 0 || game >= E.G || tree < 0 || tree >= 2) return AZ_ERR_INVALID;
  if (tree >= E.T) tree = 0;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  int32_t ti[TI_COUNT];
  const size_t gt = (size_t)game * E.T + tree;
  CUDA_CHECK(cudaMemcpy(ti, E.ti + gt * TI_COUNT, sizeof ti, cudaMemcpyDeviceToHost));
  *n_rows = 0;
  if (ti[TI_ROOT] < 0) return AZ_OK;
  const int na = ti[TI_ALLOC];
  std::vector<uint32_t> N(na), meta(na);
  std::vector<float> W(na), Pr(na);
  std::vector<int32_t> first(na);
  const size_t tb = gt * (size_t)e->P.max_nodes;
  CUDA_CHECK(cudaMemcpy(N.data(), E.N + tb, (size_t)na * 4, cudaMemcpyDeviceToHost));
  CUDA_CHECK(cudaMemcpy(W.data(), E.W + tb, (size_t)na * 4, cudaMemcpyDeviceToHost));
  CUDA_CHECK(cudaMemcpy(Pr.data(), E.Pr + tb, (size_t)na * 4, cudaMemcpyDeviceToHost));
  CUDA_CHECK(cudaMemcpy(meta.data(), E.meta + tb, (size_t)na * 4, cudaMemcpyDeviceToHost));
  CUDA_CHECK(cudaMemcpy(first.data(), E.first + tb, (size_t)na * 4, cudaMemcpyDeviceToHost));
  // iterative DFS preorder, children in list order
  std::vector<std::pair<int, int>> stack;  // (node, depth)
  stack.push_back({ti[TI_ROOT], 0});
  int cnt = 0;
  while (!stack.empty()) {
    auto [nd, dp] = stack.back();
    stack.pop_back();
    uint32_t m = meta[nd];
    int nc = META_NCHILD(m);
    if (cnt < cap_rows) {
      int32_t* r = rows + (size_t)cnt * 7;
      uint32_t wb, pb;
      memcpy(&wb, &W[nd], 4); memcpy(&pb, &Pr[nd], 4);
      r[0] = dp; r[1] = META_MOVE(m); r[2] = (int32_t)N[nd]; r[3] = (int32_t)wb; r[4] = (int32_t)pb;
      r[5] = (int32_t)META_EXPANDED(m); r[6] = nc;
    }
    cnt++;
    for (int j = nc - 1; j >= 0; j--) stack.push_back({first[nd] + j, dp + 1});
  }
  *n_rows = cnt;
  GUARD_END(e)
  return AZ_OK;
}

// ---- rules ------------------------------------------------------------------------------------
int az_rules_apply(az_engine* e, int32_t n, const int32_t* boards, const int32_t* players, const int32_t* moves,
                   int32_t* check, int32_t* applied, int32_t* out_boards, int32_t* taken) {
  if (n < 0) return AZ_ERR_INVALID;
  if (n == 0) return AZ_OK;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  const int cells = e->P.cells;
  int *d_b, *d_p, *d_m, *d_c, *d_a, *d_o, *d_t;
  CUDA_CHECK(cudaMalloc(&d_b, (size_t)n * cells * 4)); CUDA_CHECK(cudaMalloc(&d_o, (size_t)n * cells * 4));
  CUDA_CHECK(cudaMalloc(&d_p, (size_t)n * 4)); CUDA_CHECK(cudaMalloc(&d_m, (size_t)n * 4));
  CUDA_CHECK(cudaMalloc(&d_c, (size_t)n * 4)); CUDA_CHECK(cudaMalloc(&d_a, (size_t)n * 4)); CUDA_CHECK(cudaMalloc(&d_t, (size_t)n * 4));
  CUDA_CHECK(cudaMemcpy(d_b, boards, (size_t)n * cells * 4, cudaMemcpyHostToDevice));
  CUDA_CHECK(cudaMemcpy(d_p, players, (size_t)n * 4, cudaMemcpyHostToDevice));
  CUDA_CHECK(cudaMemcpy(d_m, moves, (size_t)n * 4, cudaMemcpyHostToDevice));
  launch_rules_apply(e->P, e->E.cellsP, n, d_b, d_p, d_m, d_c, d_a, d_o, d_t, e->stream); e->launches++;
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  CUDA_CHECK(cudaMemcpy(check, d_c, (size_t)n * 4, cudaMemcpyDeviceToHost));
  CUDA_CHECK(cudaMemcpy(applied, d_a, (size_t)n * 4, cudaMemcpyDeviceToHost));
  CUDA_CHECK(cudaMemcpy(taken, d_t, (size_t)n * 4, cudaMemcpyDeviceToHost));
  CUDA_CHECK(cudaMemcpy(out_boards, d_o, (size_t)n * cells * 4, cudaMemcpyDeviceToHost));
  cudaFree(d_b); cudaFree(d_o); cudaFree(d_p); cudaFree(d_m); cudaFree(d_c); cudaFree(d_a); cudaFree(d_t);
  GUARD_END(e)
  return AZ_OK;
}
int az_rules_status(az_engine* e, int32_t n, const int32_t* boards, const int32_t* passes, int32_t* ended,
                    int32_t* winner, float* score_black, float* score_white) {
  if (n < 0) return AZ_ERR_INVALID;
  if (n == 0) return AZ_OK;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  const int cells = e->P.cells;
  int *d_b, *d_p, *d_e, *d_w; float *d_sb, *d_sw;
  CUDA_CHECK(cudaMalloc(&d_b, (size_t)n * cells * 4)); CUDA_CHECK(cudaMalloc(&d_p, (size_t)n * 4));
  CUDA_CHECK(cudaMalloc(&d_e, (size_t)n * 4)); CUDA_CHECK(cudaMalloc(&d_w, (size_t)n * 4));
  CUDA_CHECK(cudaMalloc(&d_sb, (size_t)n * 4)); CUDA_CHECK(cudaMalloc(&d_sw, (size_t)n * 4));
  CUDA_CHECK(cudaMemcpy(d_b, boards, (size_t)n * cells * 4, cudaMemcpyHostToDevice));
  std::vector<int> zero(n, 0);
  CUDA_CHECK(cudaMemcpy(d_p, passes ? passes : zero.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
  launch_rules_status(e->P, e->E.cellsP, n, d_b, d_p, d_e, d_w, d_sb, d_sw, e->stream); e->launches++;
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  CUDA_CHECK(cudaMemcpy(ended, d_e, (size_t)n * 4, cudaMemcpyDeviceToHost));
  CUDA_CHECK(cudaMemcpy(winner, d_w, (size_t)n * 4, cudaMemcpyDeviceToHost));
  CUDA_CHECK(cudaMemcpy(score_black, d_sb, (size_t)n * 4, cudaMemcpyDeviceToHost));
  CUDA_CHECK(cudaMemcpy(score_white, d_sw, (size_t)n * 4, cudaMemcpyDeviceToHost));
  cudaFree(d_b); cudaFree(d_p); cudaFree(d_e); cudaFree(d_w); cudaFree(d_sb); cudaFree(d_sw);
  GUARD_END(e)
  return AZ_OK;
}

// ---- dual.Train (meta.go:16-54) and the gradient all-reduce (K7/K8) ---------------------------
static void ensure_train(az_engine* e) { train_ws_alloc(e->train, e->L); }

static void shuffle_rows(std::vector<float>& Xs, std::vector<float>& Pi, std::vector<float>& V, int rows, uint64_t* s) {
  // shuffleBatch (meta.go:57-102): Fisher-Yates over rows, j = r.Intn(i+1), injected splitmix64 stream
  const size_t xr = Xs.size() / rows, pr = Pi.size() / rows;
  for (int i = 0; i < rows; i++) {
    int j = (int)(splitmix64(s) % (uint64_t)(i + 1));
    if (i == j) continue;
    std::swap_ranges(Xs.begin() + i * xr, Xs.begin() + (i + 1) * xr, Xs.begin() + j * xr);
    std::swap_ranges(Pi.begin() + i * pr, Pi.begin() + (i + 1) * pr, Pi.begin() + j * pr);
    std::swap(V[i], V[j]);
  }
}

// one step on the batch already staged in the workspace: grads, [all-reduce], SGD
static void train_one(az_engine* e, int net, float lr) {
  train_step_grads(e->train, e->L, e->net_params[net], e->stream, &e->launches);
  if (e->p2p) {  // K8: reduce-scatter + SGD + all-gather in one kernel over NVLink peer memory
    train_allreduce_sgd_p2p(e->d_peer_grads, e->d_peer_params[net], e->d_peer_flags, e->my_flags, e->rank, e->world, e->L.total,
                            lr, ++e->epoch, e->done_counter, e->num_sms, e->E.err, e->stream, &e->launches);
    return;
  }
  float gscale = 1.0f;
  if (e->comm) {
    nccl_allreduce_sum(e, train_ws_grads(e->train), e->L.total);
    gscale = 1.0f / (float)e->world;
  }
  train_sgd(e->train, e->L, e->net_params[net], lr, gscale, e->stream, &e->launches);
}

int az_train(az_engine* e, int32_t net, float* Xs, float* Pi, float* V, int32_t batches, int32_t iterations, float lr,
             uint64_t shuffle_seed, float* costs_out) {
  if (net < 0 || net > 1 || batches < 1 || iterations < 0) return AZ_ERR_INVALID;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  ensure_train(e);
  const NetDims& d = e->L.d;
  const size_t xr = (size_t)d.F * d.HW(), pr = d.A1;
  const int rows = batches * d.B;
  std::vector<float> x(Xs, Xs + rows * xr), p(Pi, Pi + rows * pr), v(V, V + rows);
  float *dX, *dPi, *dV;
  train_ws_inputs(e->train, &dX, &dPi, &dV);
  std::vector<float> costs((size_t)batches * iterations);
  uint64_t rs = shuffle_seed;
  if (e->comm && e->world > 1) {  // every rank must run the same number of collective steps: agree before the first one
    if (!e->d_agree) e->d_agree = e->dalloc<int32_t>(2);
    int32_t* d2 = e->d_agree;
    const int32_t mine[2] = {batches * iterations, -(batches * iterations)};
    CUDA_CHECK(cudaMemcpyAsync(d2, mine, 8, cudaMemcpyHostToDevice, e->stream));
    NcclApi& na = nccl_api();
    ncclResult_t r = na.AllReduce(d2, d2, 2, ncclInt32, ncclMax, (ncclComm_t)e->comm, e->stream);
    if (r != ncclSuccess) throw std::runtime_error(std::string("ncclAllReduce(step count): ") + na.GetErrorString(r));
    int32_t got[2];
    CUDA_CHECK(cudaMemcpyAsync(got, d2, 8, cudaMemcpyDeviceToHost, e->stream));
    CUDA_CHECK(cudaStreamSynchronize(e->stream));
    if (got[0] != mine[0] || got[1] != mine[1]) throw std::runtime_error("az_train: ranks disagree on batches x iterations (data-parallel steps are collective)");
  }
  for (int it = 0; it < iterations; it++) {
    for (int bat = 0; bat < batches; bat++) {
      const size_t s0 = (size_t)bat * d.B;
      CUDA_CHECK(cudaMemcpyAsync(dX, x.data() + s0 * xr, d.B * xr * 4, cudaMemcpyHostToDevice, e->stream));
      CUDA_CHECK(cudaMemcpyAsync(dPi, p.data() + s0 * pr, d.B * pr * 4, cudaMemcpyHostToDevice, e->stream));
      CUDA_CHECK(cudaMemcpyAsync(dV, v.data() + s0, d.B * 4, cudaMemcpyHostToDevice, e->stream));
      train_one(e, net, lr);
      CUDA_CHECK(cudaMemcpyAsync(&costs[(size_t)it * batches + bat], train_ws_cost(e->train), 4, cudaMemcpyDeviceToHost, e->stream));
      CUDA_CHECK(cudaStreamSynchronize(e->stream));  // pageable staging buffers are reused next batch
      if (e->p2p) {
        int bits = 0;
        CUDA_CHECK(cudaMemcpy(&bits, e->E.err, 4, cudaMemcpyDeviceToHost));
        if (bits) { CUDA_CHECK(cudaMemset(e->E.err, 0, 4)); CUDA_CHECK(cudaMemset(e->done_counter, 0, 4)); return device_error_to_rc(e, bits); }
      }
    }
    shuffle_rows(x, p, v, rows, &rs);
  }
  memcpy(Xs, x.data(), x.size() * 4); memcpy(Pi, p.data(), p.size() * 4); memcpy(V, v.data(), v.size() * 4);
  if (costs_out) memcpy(costs_out, costs.data(), costs.size() * 4);
  GUARD_END(e)
  return AZ_OK;
}

int az_train_grads(az_engine* e, int32_t net, const float* X, const float* Pi, const float* V, float* grads_out,
                   float* cost_out) {
  if (net < 0 || net > 1) return AZ_ERR_INVALID;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  ensure_train(e);
  const NetDims& d = e->L.d;
  float *dX, *dPi, *dV;
  train_ws_inputs(e->train, &dX, &dPi, &dV);
  CUDA_CHECK(cudaMemcpyAsync(dX, X, (size_t)d.B * d.F * d.HW() * 4, cudaMemcpyHostToDevice, e->stream));
  CUDA_CHECK(cudaMemcpyAsync(dPi, Pi, (size_t)d.B * d.A1 * 4, cudaMemcpyHostToDevice, e->stream));
  CUDA_CHECK(cudaMemcpyAsync(dV, V, (size_t)d.B * 4, cudaMemcpyHostToDevice, e->stream));
  train_step_grads(e->train, e->L, e->net_params[net], e->stream, &e->launches);
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  if (grads_out) CUDA_CHECK(cudaMemcpy(grads_out, train_ws_grads(e->train), e->L.total * 4, cudaMemcpyDeviceToHost));
  if (cost_out) CUDA_CHECK(cudaMemcpy(cost_out, train_ws_cost(e->train), 4, cudaMemcpyDeviceToHost));
  GUARD_END(e)
  return AZ_OK;
}
int az_train_apply(az_engine* e, int32_t net, const float* grads, float lr) {
  if (net < 0 || net > 1) return AZ_ERR_INVALID;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  ensure_train(e);
  CUDA_CHECK(cudaMemcpyAsync(train_ws_grads(e->train), grads, e->L.total * 4, cudaMemcpyHostToDevice, e->stream));
  train_sgd(e->train, e->L, e->net_params[net], lr, 1.0f, e->stream, &e->launches);
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  GUARD_END(e)
  return AZ_OK;
}

int az_comm_unique_id(uint8_t id[128]) {
  try {
    NcclApi& n = nccl_api();
    ncclUniqueId u;
    if (n.GetUniqueId(&u) != ncclSuccess) return AZ_ERR_CUDA;
    static_assert(sizeof(u) == 128, "ncclUniqueId size");
    memcpy(id, &u, 128);
    return AZ_OK;
  } catch (const std::exception& ex) { g_create_error = ex.what(); return AZ_ERR_UNSUPPORTED; }
}
int az_comm_init(az_engine* e, int32_t rank, int32_t world, const uint8_t id[128]) {
  if (world < 1 || rank < 0 || rank >= world) return AZ_ERR_INVALID;
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  NcclApi& n = nccl_api();
  ncclUniqueId u;
  memcpy(&u, id, 128);
  ncclComm_t c;
  ncclResult_t r = n.CommInitRank(&c, world, u, rank);
  if (r != ncclSuccess) throw std::runtime_error(std::string("ncclCommInitRank: ") + n.GetErrorString(r));
  e->comm = c; e->rank = rank; e->world = world;
  // ---- peer-memory path: exchange CUDA IPC handles of {grads, params A, params B, flags} over the new communicator
  const char* mode = getenv("AZ_TRAIN_COLLECTIVE");  // "nccl" keeps the plain ncclAllReduce + SGD (A/B checks)
  if (world > 1 && !(mode && strcmp(mode, "nccl") == 0)) {
    ensure_train(e);
    CUDA_CHECK(cudaDeviceGetAttribute(&e->num_sms, cudaDevAttrMultiProcessorCount, e->device));
    e->my_flags = e->dalloc<int>(2 * world);
    e->done_counter = e->dalloc<unsigned int>(1);
    void* mine[4] = {train_ws_grads(e->train), e->net_params[0], e->net_params[1], e->my_flags};
    std::vector<cudaIpcMemHandle_t> hs((size_t)4 * world);
    for (int k = 0; k < 4; k++) CUDA_CHECK(cudaIpcGetMemHandle(&hs[(size_t)4 * rank + k], mine[k]));
    cudaIpcMemHandle_t* dh = e->dalloc<cudaIpcMemHandle_t>((size_t)4 * world);
    CUDA_CHECK(cudaMemcpy(dh + (size_t)4 * rank, &hs[(size_t)4 * rank], 4 * sizeof(cudaIpcMemHandle_t), cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaDeviceSynchronize());
    ncclResult_t ar = n.AllGather(dh + (size_t)4 * rank, dh, 4 * sizeof(cudaIpcMemHandle_t), ncclChar, c, e->stream);
    if (ar != ncclSuccess) throw std::runtime_error(std::string("ncclAllGather(ipc handles): ") + n.GetErrorString(ar));
    CUDA_CHECK(cudaStreamSynchronize(e->stream));
    CUDA_CHECK(cudaMemcpy(hs.data(), dh, hs.size() * sizeof(cudaIpcMemHandle_t), cudaMemcpyDeviceToHost));
    std::vector<float*> pg(world), pa(world), pb(world);
    std::vector<int*> pf(world);
    for (int r2 = 0; r2 < world; r2++) {
      void* ptr[4];
      for (int k = 0; k < 4; k++) {
        if (r2 == rank) { ptr[k] = mine[k]; continue; }
        CUDA_CHECK(cudaIpcOpenMemHandle(&ptr[k], hs[(size_t)4 * r2 + k], cudaIpcMemLazyEnablePeerAccess));
        e->ipc_opened.push_back(ptr[k]);
      }
      pg[r2] = (float*)ptr[0]; pa[r2] = (float*)ptr[1]; pb[r2] = (float*)ptr[2]; pf[r2] = (int*)ptr[3];
    }
    e->d_peer_grads = e->dalloc<float*>(world); e->d_peer_params[0] = e->dalloc<float*>(world);
    e->d_peer_params[1] = e->dalloc<float*>(world); e->d_peer_flags = e->dalloc<int*>(world);
    CUDA_CHECK(cudaMemcpy(e->d_peer_grads, pg.data(), world * sizeof(void*), cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(e->d_peer_params[0], pa.data(), world * sizeof(void*), cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(e->d_peer_params[1], pb.data(), world * sizeof(void*), cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(e->d_peer_flags, pf.data(), world * sizeof(void*), cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaDeviceSynchronize());
    e->p2p = true;
  }
  GUARD_END(e)
  return AZ_OK;
}

int az_comm_bench(az_engine* e, int32_t net, int32_t iters, double* ms_out, double* bytes_out) {
  if (net < 0 || net > 1 || iters < 1) return AZ_ERR_INVALID;
  if (!e->comm) { e->err = "az_comm_bench: no communicator"; return AZ_ERR_STATE; }
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  ensure_train(e);
  cudaEvent_t a, b;
  CUDA_CHECK(cudaEventCreate(&a)); CUDA_CHECK(cudaEventCreate(&b));
  auto step = [&]() {
    if (e->p2p) train_allreduce_sgd_p2p(e->d_peer_grads, e->d_peer_params[net], e->d_peer_flags, e->my_flags, e->rank, e->world,
                                        e->L.total, 0.0f, ++e->epoch, e->done_counter, e->num_sms, e->E.err, e->stream, &e->launches);
    else { nccl_allreduce_sum(e, train_ws_grads(e->train), e->L.total); train_sgd(e->train, e->L, e->net_params[net], 0.0f, 1.0f, e->stream, &e->launches); }
  };
  for (int i = 0; i < 2; i++) step();  // warm-up
  CUDA_CHECK(cudaEventRecord(a, e->stream));
  for (int i = 0; i < iters; i++) step();
  CUDA_CHECK(cudaEventRecord(b, e->stream));
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  float ms = 0;
  CUDA_CHECK(cudaEventElapsedTime(&ms, a, b));
  cudaEventDestroy(a); cudaEventDestroy(b);
  if (ms_out) *ms_out = ms / iters;
  if (bytes_out) *bytes_out = 2.0 * (e->world - 1) / e->world * (double)e->L.total * 4.0;
  if (e->p2p) {
    int bits = 0;
    CUDA_CHECK(cudaMemcpy(&bits, e->E.err, 4, cudaMemcpyDeviceToHost));
    if (bits) { CUDA_CHECK(cudaMemset(e->E.err, 0, 4)); CUDA_CHECK(cudaMemset(e->done_counter, 0, 4)); return device_error_to_rc(e, bits); }
  }
  GUARD_END(e)
  return AZ_OK;
}

int az_profile(az_engine* e, int32_t enable, double out[8]) {
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  if (!e->prof_start) { CUDA_CHECK(cudaEventCreate(&e->prof_start)); CUDA_CHECK(cudaEventCreate(&e->prof_stop)); }
  if (out) {
    for (int i = 0; i < 8; i++) out[i] = 0;
    if (e->use_tc) for (int a = 0; a < 2; a++) tc_tower_profile_collect(e->tc[a], e->stream, &out[0], &out[1], &out[2], &out[3]);
    out[5] = e->use_tc ? (double)tc_tower_kernel_kind(e->tc[0]) : -1.0;  // which kernel runs the fused layers
    if ((e->profiling || e->prof_region) && !enable) {  // whole region on the engine's stream, device-timed
      CUDA_CHECK(cudaEventRecord(e->prof_stop, e->stream));
      CUDA_CHECK(cudaEventSynchronize(e->prof_stop));
      float ms = 0;
      CUDA_CHECK(cudaEventElapsedTime(&ms, e->prof_start, e->prof_stop));
      out[4] = ms;
    }
  }
  if (enable) { CUDA_CHECK(cudaStreamSynchronize(e->stream)); CUDA_CHECK(cudaEventRecord(e->prof_start, e->stream)); }
  if (e->use_tc) for (int a = 0; a < 2; a++) tc_tower_profile(e->tc[a], enable == 1);
  e->profiling = enable == 1;    // event records inside the wave: replay the plain launch sequence instead of the graph
  e->prof_region = enable == 2;  // region timing only: the captured wave graph keeps running
  GUARD_END(e)
  return AZ_OK;
}

int az_counters_get(const az_engine* ce, az_counters* out) {
  az_engine* e = const_cast<az_engine*>(ce);
  memset(out, 0, sizeof *out);
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  unsigned long long c[CNT_COUNT];
  CUDA_CHECK(cudaMemcpy(c, e->E.counters, sizeof c, cudaMemcpyDeviceToHost));
  out->searches = c[CNT_SEARCHES]; out->sims = c[CNT_SIMS]; out->null_results = c[CNT_NULL]; out->evals = c[CNT_EVALS];
  out->select_children = c[CNT_SEL_CHILDREN]; out->select_levels = c[CNT_SEL_LEVELS]; out->created = c[CNT_CREATED];
  out->backup_nodes = c[CNT_BACKUP]; out->kernel_launches = e->launches;
  GUARD_END(e)
  return AZ_OK;
}
int az_counters_reset(az_engine* e) {
  GUARD_BEGIN
  CUDA_CHECK(cudaSetDevice(e->device));
  CUDA_CHECK(cudaStreamSynchronize(e->stream));
  CUDA_CHECK(cudaMemset(e->E.counters, 0, CNT_COUNT * sizeof(unsigned long long)));
  e->launches = 0;
  GUARD_END(e)
  return AZ_OK;
}

}  // extern "C"
