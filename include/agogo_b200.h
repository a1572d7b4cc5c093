/*
 * agogo_b200.h — C ABI of the H100-native AlphaZero self-play engine that slots under
 * gorgonia/agogo's Go API (AZ / Agent / Arena, game.State, mcts.Config, dual.Config).
 *
 * The reference has no FFI boundary (one Go process, Go interfaces only); every entry point
 * below names the Go seam it replaces (file:line relative to the reference tree) and is what a
 * cgo shim binds (see INTEGRATION.md and go/ for the stub).  Plain pointers and sizes only:
 * caller allocates every in/out buffer, the engine copies before returning and never retains a
 * caller pointer (cgo rule).  One in-flight mutating call per engine handle; az_infer may be
 * called concurrently with nothing else.  Every function returns 0 on success or a negative
 * AZ_ERR_* code; az_last_error() gives the message.  Where the reference panics (agogo.go:42-47
 * invalid config, agent.go:66-71 inference error, node.go:232-234 "Cannot return nil") the
 * engine returns AZ_ERR_PANIC and the Go shim re-panics.
 *
 * Two libraries export exactly these symbols:
 *   agogo_b200/libagogo_b200.so   the product: hand-written sm_90a CUDA, fails loudly without a GPU
 *   oracle/libazoracle.so         TEST INFRASTRUCTURE: CPU restatement of the reference algorithm
 */
#ifndef AGOGO_B200_H
#define AGOGO_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AZ_OK 0
#define AZ_ERR_INVALID (-1)  /* bad argument / invalid config */
#define AZ_ERR_CUDA (-2)     /* CUDA runtime/driver failure (no GPU, OOM, launch error) */
#define AZ_ERR_PANIC (-3)    /* a condition on which the reference panics */
#define AZ_ERR_UNSUPPORTED (-4)
#define AZ_ERR_STATE (-5)    /* call sequence violation */

/* game/state.go:9-13 */
#define AZ_NONE 0
#define AZ_BLACK 1
#define AZ_WHITE 2
/* mcts/mcts.go:20-23 */
#define AZ_PASS (-1)
#define AZ_RESIGN (-2)

enum az_game_kind { AZ_GAME_MNK = 0 /* game/mnk */, AZ_GAME_C4 = 1 /* game/c4 */, AZ_GAME_WQ = 2 /* game/wq */ };
enum az_encoder_kind {
  AZ_ENC_TWO_PLANE = 0, /* cmd/tictactoe/main.go:26-47 */
  AZ_ENC_WQ18 = 1       /* encoding_helper.go:29-68 (WQEncoder) */
};
enum az_inferer_kind {
  AZ_INF_DUAL = 0,  /* dual.Infer snapshot of the agent's net (agent.go:42-57, meta.go:125-190) */
  AZ_INF_DUMMY = 1, /* dummy.go: uniform 1/ActionSpace policy of length ActionSpace, value by colour */
  AZ_INF_TABLE = 2  /* scripted policy/value rows keyed by MoveNumber (mcts/example_test.go:38-72) */
};

/* game constructors: mnk.New(m,n,k) mnk.go:35; c4.New(rows,cols,N) c4/game.go:24; wq.New(size,0,komi) wq/game.go:26.
 * max_moves (0 = none) and zobrist_seed are engine-side completions: the reference has no move
 * cap and seeds its Zobrist table from the clock (wq/zobrist.go:32). */
typedef struct az_game_desc {
  int32_t kind;
  int32_t m, n, k; /* mnk: m,n,k; c4: rows,cols,N-to-win; wq: m=n=board size, k unused */
  float komi;
  int32_t max_moves;
  uint64_t zobrist_seed;
} az_game_desc;

/* mcts.Config, mcts/tree.go:15-29, field for field; `sims` is new: the fixed number of
 * pipeline iterations per Search (the reference stops on Timeout only, search.go:133).
 * `workers` is the number of concurrent pipeline calls per tree — the reference starts
 * runtime.NumCPU() searchStates (search.go:112-130) whose interleaving Go leaves unspecified;
 * here they run under one fixed schedule: rounds of `workers` descents that each set the
 * virtual-loss flag on their path (search.go:222) and stop at the leaf they want evaluated, ONE
 * batched inference for the round, then expansion + Update + undoVirtualLoss in start order.
 * 0 or 1 = the canonical single worker (bit-exact tree for a given seed); > 1 multiplies the
 * evaluation batch of a single position by `workers` (Agent.Search on one state, GTP play). */
typedef struct az_mcts_config {
  float puct;
  int64_t timeout_ns;
  int32_t m, n;
  int32_t random_count;
  int32_t budget;
  uint32_t random_min_visits;
  float random_temperature;
  int32_t dumb_pass;
  float resign_percentage;
  int32_t pass_preference; /* mcts/mcts.go:31-38 */
  int32_t sims;
  int32_t workers;
} az_mcts_config;

/* dual.Config, dualnet/config.go:4-16, field for field. */
typedef struct az_dual_config {
  int32_t k, shared_layers, fc;
  double l2;
  int32_t batch_size, width, height, features;
  int32_t action_space;
  int32_t fwd_only;
} az_dual_config;

#define AZ_FLAG_SHARED_TREE 1u /* one MCTS searched by both colours (mcts/example_test.go:74-156) */
#define AZ_FLAG_FP32_TOWER 2u  /* force the fp32 CUDA-core tower (validation kernel) instead of the tensor cores */
/* Precision policy of the tensor-core tower: fp32-faithful — fp16 hi/lo operand split, three tensor passes per MAC,
 * policy/value within 1e-4 of the fp32 forward (DESIGN.md section 4).  AZ_FLAG_FAST_TOWER is accepted for a faster,
 * less precise tower; this build has no such kernel and runs the three passes for it too. */
#define AZ_FLAG_FAST_TOWER 4u
/* wq only — OUR completion of the reference's unfinished Go rules (SURVEY section 8f row 4), off by default (the default
 * keeps wq.Game exactly as written: occupied points "legal", no ko, the row-0 flood-fill Score).  With the flag:
 * occupied points and true suicide are illegal, simple ko AND positional superko (game.go:77's TODO: no move may recreate
 * the stones of an earlier position of the game — inside the search: of the game or of the descent; for az_search on a
 * caller-owned position: of the earlier boards in az_state.hist), own single-point eyes are never filled (the
 * "eye-ish situations" noPass expects Check to reject, search.go:543), Score = area (stones + empty regions touching one colour
 * only) and Ended adds komi to White.  Same arithmetic everywhere else; engine and oracle are compared bit for bit under
 * the flag too. */
#define AZ_FLAG_WQ_COMPLETE 8u

typedef struct az_engine_desc {
  az_game_desc game;
  az_mcts_config mcts;
  az_dual_config nn;
  int32_t encoder;  /* az_encoder_kind (agogo.Config.Encoder, datatypes.go:22) */
  int32_t n_games;  /* concurrent Arena games resident on the device */
  int32_t device;   /* CUDA device ordinal */
  uint32_t flags;
  uint64_t seed;    /* replaces the reference's time.Now() seeds (arena.go:61, tree.go:84) */
  int32_t act_scale_log2;     /* tensor-core tower: activations are stored as fp16 hi/lo of x*2^this; 0 = default (-2: |x| up to 2.6e5
                               * before AZ_ERR_PANIC "activation overflow"; between -5 and 5 the outputs agree to the storage's
                               * resolution: |x| below 2^-(3+this) is kept to an absolute 2^-(25+this)) */
  int32_t max_nodes_per_tree; /* 0 = derive from sims and action space */
} az_engine_desc;

typedef struct az_engine az_engine;

/* agogo.New (agogo.go:41-73) + MakeArena (arena.go:42-71): validates both configs (the
 * reference panics), allocates nets A and B, game slots, trees.  Nets are NOT initialised. */
int az_engine_create(const az_engine_desc* desc, az_engine** out);
void az_engine_destroy(az_engine* e);
const char* az_last_error(const az_engine* e); /* e may be NULL: error of the last failed create */

/* ---- networks: slot 0 = Agent A's NN, slot 1 = Agent B's NN ---------------------------------- */
/* dual.Model() (dual.go:134-142): tensors in graph-creation order, training shapes. */
int az_net_param_count(const az_engine* e, int32_t* n_tensors, uint64_t* n_floats);
int az_net_param_desc(const az_engine* e, int32_t i, char name[96], int32_t shape[4], int32_t* rank,
                      uint64_t* offset, uint64_t* size);
int az_net_init(az_engine* e, int32_t net, uint64_t seed);                  /* dual.New+Init, dual.go:33-48 */
int az_net_get_params(az_engine* e, int32_t net, float* out, uint64_t n);   /* GobEncode payload, dual.go:180-190 */
int az_net_set_params(az_engine* e, int32_t net, const float* in, uint64_t n); /* GobDecode, dual.go:192-206 */
int az_net_copy(az_engine* e, int32_t dst, int32_t src);                    /* A.NN = B.NN, agogo.go:161 */

/* ---- agents: 0 = A, 1 = B -------------------------------------------------------------------- */
/* Agent.SwitchToInference (agent.go:42-57) / Agent.useDummy (agent.go:105-113).  For
 * AZ_INF_DUMMY `dummy_player` is the Agent.Player captured when useDummy ran. */
int az_agent_set_inferer(az_engine* e, int32_t agent, int32_t kind, int32_t dummy_player);
int az_agent_set_table(az_engine* e, int32_t agent, int32_t n_rows, int32_t row_len, const float* policy_rows,
                       const float* values);
/* Agent.NNOutput / Inferer.Infer (agent.go:83-89, meta.go:168-190) batched: planes [n,F,H,W]
 * -> policy [n,action_space], value [n].  Uses the agent's inference snapshot. */
int az_infer(az_engine* e, int32_t agent, const float* planes, int32_t n, float* policy, float* value);
/* Diagnostics: the same forward as az_infer, but returns the residual tower's output — the activations the policy and value
 * head convs read — as fp32 tower_out [n,K,H,W].  On the tensor-core tower that is the stored fp16 hi/lo pair,
 * (hi + lo) / 2^act_scale_log2.  Lets a test compare one conv layer at a time: a net with SharedLayers = l computes the
 * first l blocks of a deeper net with the same leading weights. */
int az_infer_tower(az_engine* e, int32_t agent, const float* planes, int32_t n, float* tower_out);
int az_agent_stats(const az_engine* e, int32_t agent, float* wins, float* loss, float* draw);
int az_agent_reset_stats(az_engine* e, int32_t agent); /* agent.go:115-121 */

/* ---- Arena.Play (arena.go:80-179) over many concurrent games --------------------------------- */
/* az_arena_play == `n_games` sequential Arena.Play(record, nil, nil) calls, each followed by
 * game.Reset() (agogo.go:93-97,144-148), run concurrently on the device.  Game i takes the i-th
 * next draw of the arena coin RNG.  Recorded examples are appended to the engine's example list
 * in game order, then ply order. */
int az_arena_play(az_engine* e, int32_t n_games, int32_t record);
/* the same, one ply at a time (tests, bench): begin -> step* -> finish */
int az_arena_begin(az_engine* e, int32_t n_games, int32_t record);
int az_arena_step(az_engine* e, int32_t* n_active); /* Search + Apply for every unfinished game */
int az_arena_finish(az_engine* e);                  /* labels, win/loss/draw, fresh trees */
/* finer still: one MCTS.Search (search.go:92-164) split into its phases for every active game */
int az_search_begin(az_engine* e);                   /* updateRoot + prepareRoot (1 evaluation) */
int az_search_run(az_engine* e, int32_t n_iterations); /* n x pipeline (search.go:209-257) per game */
int az_search_end(az_engine* e);                     /* bestMove, example, Apply, switchPlayer */

/* Agent.Search on an EXTERNAL position (agent.go:77-80: MCTS.SetGame(g); MCTS.Search(a.Player)) — the
 * README's inference use.  The Go shim marshals game.State getters into az_state: Board(), ToMove(),
 * MoveNumber(), Passes(), for the WQEncoder Historical(MoveNumber-n_hist .. MoveNumber-1), and the tail of the
 * state's move history (what UndoLastMove / Fwd walk).  Returns the chosen move and, optionally, the root children's
 * visit counts indexed by move (Pass at index ActionSpace).  Not callable while an arena is running; uses game slot 0.
 *
 * Tree reuse (updateRoot / newRootState, search.go:424-500): the agent's tree survives the call, as the Agent's MCTS
 * does in the reference.  The next az_search of the same agent re-roots it when the new position continues the one
 * searched last: d = MoveNumber - prev.MoveNumber >= 0, the last d entries of `moves` undone from the board give the
 * previous board (State.Eq), and each of those moves is a child of the successive roots (findChild); the siblings'
 * subtrees become unreachable (cleanup), the pool keeps growing until az_agent_reset_tree.  Anything else — no move
 * list, a different line of play, a missing child — searches a brand-new root, exactly as the reference falls back to
 * New(Pass|first legal move).  Reuse can only succeed for mnk: c4's Clone pads its history (c4/game.go:142-160) and
 * wq has no UndoLastMove (wq/game.go:119), so those games always take the fresh-root path (and their pool is recycled).
 * az_arena_begin and az_agent_reset_tree (MCTS.Reset, tree.go:249-276) drop the external trees. */
typedef struct az_state {
  const int32_t* board; /* [m*n] colours */
  int32_t to_move, move_number, passes;
  int32_t last_move;    /* LastMove().Single; AZ_PASS for an empty history (mnk.go:84-89) */
  int32_t n_hist;       /* 0..8; under AZ_FLAG_WQ_COMPLETE up to the whole game (the encoder reads the last 8, superko all) */
  const int32_t* hist;  /* [n_hist][m*n], oldest first (wq18 planes; under AZ_FLAG_WQ_COMPLETE also the positions superko bars) */
  int32_t n_moves;      /* entries of `moves` (0 = history unknown: no reuse across calls) */
  const int32_t* moves; /* [n_moves][2] = (player, move), oldest first: the tail of the State's history */
  int32_t ko;           /* AZ_FLAG_WQ_COMPLETE only: the point barred by simple ko for the side to move, or -1 (0 is a point: set it) */
} az_state;
int az_search(az_engine* e, int32_t agent, const az_state* s, int32_t player, int32_t* best, float* child_visits);
int az_agent_reset_tree(az_engine* e, int32_t agent);

/* per-game results of the last begin..finish: moves played, winner (AZ_NONE/BLACK/WHITE),
 * colour of agent A, number of examples kept */
int az_game_record(const az_engine* e, int32_t game, int32_t* moves, int32_t cap, int32_t* n_moves,
                   int32_t* winner, int32_t* a_player, int32_t* n_examples);
/* game.State getters of game slot `game` (Board/ToMove/MoveNumber/Passes/Ended, state.go:125-156) */
int az_game_state(const az_engine* e, int32_t game, int32_t* board, int32_t cap, int32_t* to_move,
                  int32_t* move_number, int32_t* passes, int32_t* ended, int32_t* winner);
/* Example list (datatypes.go:38-42): boards [n,F*H*W], policies [n,A+1], values [n] */
int az_examples_count(const az_engine* e, int64_t* n);
int az_examples_read(const az_engine* e, int64_t start, int64_t n, float* boards, float* policies, float* values);
int az_examples_clear(az_engine* e);

/* canonical dump of a search tree (DFS preorder, children in list order): rows of 7 int32
 * {depth, move, visits, W bits, P bits, expanded, n_children}.  tree = agent index (0 with
 * AZ_FLAG_SHARED_TREE).  Valid between az_search_end/az_arena_step and the next search. */
int az_tree_dump(const az_engine* e, int32_t game, int32_t tree, int32_t* rows, int32_t cap_rows, int32_t* n_rows);

/* ---- rules, stateless and batched (game/mnk, game/c4, game/wq `__device__` twins) ------------ */
/* For each of n positions (board [cells] int32 colours, mover, move):
 *   check[i]    = State.Check(PlayerMove)                      (mnk.go:96, c4/game.go:53, wq/game.go:65)
 *   applied[i]  = whether the board-level Apply succeeded      (wq.go:141 Board.Apply error == nil, ...)
 *   out_boards  = board after State.Apply                      (unchanged when not applied)
 *   taken[i]    = wq: byte(len(captures)), duplicates included (wq.go:170); else 0 */
int az_rules_apply(az_engine* e, int32_t n, const int32_t* boards, const int32_t* players, const int32_t* moves,
                   int32_t* check, int32_t* applied, int32_t* out_boards, int32_t* taken);
/* ended/winner as State.Ended with passes given (mnk.go:156, c4/game.go:161, wq/game.go:94);
 * score_black/score_white = State.Score (wq: Board.Score as implemented, wq.go:173-202) */
int az_rules_status(az_engine* e, int32_t n, const int32_t* boards, const int32_t* passes, int32_t* ended,
                    int32_t* winner, float* score_black, float* score_white);

/* ---- dual.Train (dualnet/meta.go:16-54) ------------------------------------------------------ */
/* Xs [batches*batch_size, F,H,W], Pi [.., action_space], V [..]; vanilla SGD lr (reference 0.1);
 * rows are reshuffled after every pass with the injected seed (meta.go:47,57-102); costs_out
 * (may be NULL) receives batches*iterations costs.  Xs/Pi/V are shuffled in place like the
 * reference's tensors.  Gradients are all-reduced over the communicator when one is set. */
int az_train(az_engine* e, int32_t net, float* Xs, float* Pi, float* V, int32_t batches, int32_t iterations,
             float lr, uint64_t shuffle_seed, float* costs_out);

/* One Train step split at the solver boundary (meta.go:36-41: RunAll, then solver.Step): gradients
 * of one batch of exactly batch_size samples for every Model() tensor, flat in Model() order, and
 * their application w -= lr * g.  Lets a host all-reduce the gradients itself (the gloo tests do). */
int az_train_grads(az_engine* e, int32_t net, const float* X, const float* Pi, const float* V, float* grads_out,
                   float* cost_out);
int az_train_apply(az_engine* e, int32_t net, const float* grads, float lr);

/* ---- multi-GPU: gradient all-reduce only (SURVEY.md §8e) --------------------------------------
 * az_comm_init joins an NCCL communicator (one rank per GPU/process; id from az_comm_unique_id on
 * rank 0, distributed by the host).  With a communicator, every az_train step all-reduces (sum)
 * the flat gradient buffer over NVLink and applies w -= lr * g / world, so replicas stay identical;
 * every rank must call az_train with the same batches/iterations. */
int az_comm_unique_id(uint8_t id[128]);
int az_comm_init(az_engine* e, int32_t rank, int32_t world, const uint8_t id[128]);
/* Times the gradient exchange + solver step alone (lr = 0: parameters unchanged), `iters` back-to-back
 * launches with CUDA events on the engine's stream; every rank must call it.  ms_out = average per step,
 * bytes_out = bytes entering (= leaving) this rank over NVLink per step: (R-1)/R*|theta|*4 of gradient
 * reads plus the same amount of parameter writes = 2*(R-1)/R*|theta|*4 PER DIRECTION.  For the K8 roofline. */
int az_comm_bench(az_engine* e, int32_t net, int32_t iters, double* ms_out, double* bytes_out);

/* ---- counters (per engine, since create or az_counters_reset) -------------------------------- */
typedef struct az_counters {
  uint64_t searches, sims, null_results, evals;
  uint64_t select_children, select_levels, created, backup_nodes; /* HBM-byte accounting, SURVEY §8d */
  uint64_t kernel_launches; /* engine's own kernels launched (0 for the oracle) */
  uint64_t reserved[7];
} az_counters;
int az_counters_get(const az_engine* e, az_counters* out);
int az_counters_reset(az_engine* e);

/* Kernel timing for bench.py's roofline line: CUDA events on the engine's own stream around every
 * launch of the dominant kernel (the fused 3x3 conv of a residual block).  enable=1 starts a fresh
 * measurement, enable=0 stops; out (may be NULL) receives {conv_ms_total, conv_launches,
 * forward_ms_total, forward_calls, region_ms, kernel_kind, 0...} accumulated since the last enable=1; region_ms is the
 * device time between the enable=1 and the enable=0 call on the engine's stream; kernel_kind names the kernel that runs
 * the fused layers (0 k_conv3x3_tc, wgmma, three fp16 passes; 5 k_net_small; -1 fp32 tower).  enable=2 times the region only (region_ms): no per-launch events, so
 * the captured wave graph keeps running — what a launch-bound small-net workload should be timed with. */
int az_profile(az_engine* e, int32_t enable, double out[8]);

const char* az_build_info(void); /* "agogo_b200 <ver> sm_90a ..." or "oracle ..." */

#ifdef __cplusplus
}
#endif
#endif
