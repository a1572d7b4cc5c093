// agogo_b200 — common device/host definitions.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#define AZ_WARP 32
#define FULL 0xffffffffu

enum { KIND_MNK = 0, KIND_C4 = 1, KIND_WQ = 2 };
enum { C_NONE = 0, C_BLACK = 1, C_WHITE = 2 };
enum { MV_PASS = -1, MV_RESIGN = -2 };

// Device error bits, OR-ed into EngineDev::err (each maps to a reference panic or an engine limit).
enum {
  ERR_NO_ACTIVE_CHILD = 1,   // node.go:232-234 panic("Cannot return nil")
  ERR_POOL_EXHAUSTED = 2,    // node pool of a tree is full
  ERR_ROOT_NO_CHILDREN = 4,  // search.go:141-149 fallback path (not implemented on device)
  ERR_ACT_OVERFLOW = 8,      // tensor-core tower: fp16 activation overflow (raise act_scale headroom)
  ERR_NAN_PRIOR = 16,        // NaN prior reached the sort (Go's sort order is unspecified there)
  ERR_PATH_OVERFLOW = 32,
  ERR_RESIGN_APPLIED = 64,   // Arena applies Resign: every game.State.Apply indexes board[-2] and panics
  ERR_COMM_TIMEOUT = 128,    // K8: a peer never published its epoch flag (rank died / different batch count / not called collectively)
};

// Game + search parameters, passed by value to every kernel.
struct GameP {
  int kind, m, n, k;  // mnk: m,n,k ; c4: rows,cols,N ; wq: m=n=size
  int cells;          // m*n
  int A;              // State.ActionSpace(): cells, or cols for c4
  float komi;
  int max_moves;      // 0 = none
  int maxDepth;       // mcts.Config.M * N (search.go:119)
  float puct;
  int sims;
  int dont_prefer_pass;
  int dumb_pass, dont_resign;  // mcts.Config.DumbPass, PassPreference == DontResign
  float resign_pct;            // mcts.Config.ResignPercentage
  int random_count;            // mcts.Config.RandomCount / RandomMinVisits / RandomTemperature (tree.go:212-247)
  unsigned random_min_visits;
  float random_temperature;
  int shared_tree;
  int encoder;        // 0 two-plane, 1 wq18
  int F;              // feature planes
  int plane;          // F*cells
  int hist_len;       // 8 for wq18, else 0
  int max_nodes;      // per tree
  int max_plies;      // capacity of per-game move lists
  int wq_complete;    // AZ_FLAG_WQ_COMPLETE: OUR completion of the wq rules (occupied / suicide / ko + positional superko / eyes / area scoring)
};

__host__ __device__ inline int opp(int p) { return p == C_BLACK ? C_WHITE : C_BLACK; }

#define CUDA_CHECK(x)                                                                      \
  do {                                                                                     \
    cudaError_t _e = (x);                                                                  \
    if (_e != cudaSuccess) throw CudaError(_e, #x, __FILE__, __LINE__);                    \
  } while (0)

// after every <<<>>>: a bad launch configuration (grid wrap, missing shared-memory opt-in) is reported only by
// cudaGetLastError — later synchronisations return success.  cudaPeekAtLastError is legal during stream capture.
#define LAUNCH_CHECK()                                                                     \
  do {                                                                                     \
    cudaError_t _e = cudaPeekAtLastError();                                                \
    if (_e != cudaSuccess) { cudaGetLastError(); throw CudaError(_e, "kernel launch", __FILE__, __LINE__); } \
  } while (0)

struct CudaError {
  cudaError_t code;
  std::string msg;
  CudaError(cudaError_t c, const char* what, const char* file, int line) : code(c) {
    msg = std::string(cudaGetErrorString(c)) + " at " + file + ":" + std::to_string(line) + " (" + what + ")";
  }
};
