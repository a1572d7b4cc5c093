// ORACLE — TEST INFRASTRUCTURE ONLY (see game.hpp).
// Exports the same C ABI as the product library (include/agogo_b200.h) on top of the CPU
// restatement, so tests can diff the two libraries call for call.  n_games "concurrent" games are
// n independent Arena slots stepped in lockstep; each is exactly one reference Arena.Play.
#include <cstdio>
#include <cstring>
#include <exception>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "../include/agogo_b200.h"
#include "arena.hpp"

using namespace oracle;

static thread_local std::string g_create_error;

struct az_engine {
  az_engine_desc d;
  MCTSConfig mc;
  DualConfig dc;
  std::shared_ptr<Dual> nets[2];
  std::shared_ptr<Inferer> inferers[2];
  float wins[2] = {0, 0}, loss[2] = {0, 0}, draw[2] = {0, 0};
  Rng coin{0};
  uint64_t games_started = 0;
  std::vector<std::unique_ptr<Arena>> slots;
  int n_active_games = 0;  // games in the current begin..finish
  bool in_play = false, record = false;
  std::vector<Example> examples;
  std::vector<GameRecord> records;
  Counters base;  // counters accumulated from finished slots
  // Agent.Search on external positions: the Agent and its MCTS persist across az_search calls (agent.go:14-30)
  std::unique_ptr<Agent> ext_agent[2];
  bool ext_valid[2] = {false, false};
  int ext_prev_mn[2] = {0, 0};
  std::vector<int32_t> ext_prev_board[2];
  mutable std::string err;
};

static State* make_state(const az_game_desc& g, uint32_t flags = 0) {
  switch (g.kind) {
    case AZ_GAME_MNK: return new MNK(g.m, g.n, g.k);
    case AZ_GAME_C4: return new C4(g.m, g.n, g.k);
    case AZ_GAME_WQ: { WQ* w = new WQ(g.m, 0, g.komi, g.zobrist_seed); w->complete = (flags & AZ_FLAG_WQ_COMPLETE) != 0; return w; }
  }
  throw std::runtime_error("unknown game kind");
}

#define GUARD_BEGIN try {
#define GUARD_END(e)                                                       \
  }                                                                        \
  catch (const std::exception& ex) {                                       \
    (e)->err = ex.what();                                                  \
    return strstr(ex.what(), "invalid") ? AZ_ERR_INVALID : AZ_ERR_PANIC;   \
  }

extern "C" {

int az_engine_create(const az_engine_desc* desc, az_engine** out) {
  if (!desc || !out) { g_create_error = "null argument"; return AZ_ERR_INVALID; }
  try {
    std::unique_ptr<az_engine> e(new az_engine);
    e->d = *desc;
    const az_mcts_config& m = desc->mcts;
    e->mc.PUCT = m.puct; e->mc.Timeout = m.timeout_ns; e->mc.M = m.m; e->mc.N = m.n;
    e->mc.RandomCount = m.random_count; e->mc.Budget = m.budget; e->mc.RandomMinVisits = m.random_min_visits;
    e->mc.RandomTemperature = m.random_temperature; e->mc.DumbPass = m.dumb_pass != 0;
    e->mc.ResignPercentage = m.resign_percentage; e->mc.PassPref = m.pass_preference; e->mc.Sims = m.sims; e->mc.Workers = m.workers > 1 ? m.workers : 1;
    const az_dual_config& n = desc->nn;
    e->dc.K = n.k; e->dc.SharedLayers = n.shared_layers; e->dc.FC = n.fc; e->dc.L2 = n.l2;
    e->dc.BatchSize = n.batch_size; e->dc.Width = n.width; e->dc.Height = n.height; e->dc.Features = n.features;
    e->dc.ActionSpace = n.action_space; e->dc.FwdOnly = n.fwd_only != 0;
    if (!e->dc.IsValid()) { g_create_error = "NNConf is not valid. Unable to proceed"; return AZ_ERR_INVALID; }
    if (!e->mc.IsValid()) { g_create_error = "MCTSConf is not valid. Unable to proceed"; return AZ_ERR_INVALID; }
    if (desc->n_games < 1) { g_create_error = "n_games must be >= 1"; return AZ_ERR_INVALID; }
    std::unique_ptr<State> probe(make_state(desc->game, desc->flags));
    e->nets[0] = std::make_shared<Dual>(e->dc);
    e->nets[1] = std::make_shared<Dual>(e->dc);
    e->coin = Rng(derive_seed(desc->seed, 0));
    *out = e.release();
    return AZ_OK;
  } catch (const std::exception& ex) {
    g_create_error = ex.what();
    return AZ_ERR_INVALID;
  }
}
void az_engine_destroy(az_engine* e) { delete e; }
const char* az_last_error(const az_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }
const char* az_build_info(void) { return "oracle (CPU restatement of gorgonia/agogo @ b63af92; test infrastructure)"; }

int az_net_param_count(const az_engine* e, int32_t* n_tensors, uint64_t* n_floats) {
  if (n_tensors) *n_tensors = (int32_t)e->nets[0]->desc.size();
  if (n_floats) *n_floats = e->nets[0]->params.size();
  return AZ_OK;
}
int az_net_param_desc(const az_engine* e, int32_t i, char name[96], int32_t shape[4], int32_t* rank, uint64_t* offset,
                      uint64_t* size) {
  if (i < 0 || i >= (int)e->nets[0]->desc.size()) return AZ_ERR_INVALID;
  const ParamDesc& d = e->nets[0]->desc[i];
  if (name) { snprintf(name, 96, "%s", d.name.c_str()); }
  if (shape) for (int k = 0; k < 4; k++) shape[k] = d.shape[k];
  if (rank) *rank = d.rank;
  if (offset) *offset = d.offset;
  if (size) *size = d.size;
  return AZ_OK;
}
int az_net_init(az_engine* e, int32_t net, uint64_t seed) {
  if (net < 0 || net > 1) return AZ_ERR_INVALID;
  e->nets[net] = std::make_shared<Dual>(e->dc);
  e->nets[net]->Init(seed);
  return AZ_OK;
}
int az_net_get_params(az_engine* e, int32_t net, float* out, uint64_t n) {
  if (net < 0 || net > 1 || n != e->nets[net]->params.size()) return AZ_ERR_INVALID;
  memcpy(out, e->nets[net]->params.data(), n * 4);
  return AZ_OK;
}
int az_net_set_params(az_engine* e, int32_t net, const float* in, uint64_t n) {
  if (net < 0 || net > 1 || n != e->nets[net]->params.size()) return AZ_ERR_INVALID;
  memcpy(e->nets[net]->params.data(), in, n * 4);
  return AZ_OK;
}
int az_net_copy(az_engine* e, int32_t dst, int32_t src) {
  if (dst < 0 || dst > 1 || src < 0 || src > 1) return AZ_ERR_INVALID;
  e->nets[dst] = std::make_shared<Dual>(*e->nets[src]);
  return AZ_OK;
}

int az_agent_set_inferer(az_engine* e, int32_t agent, int32_t kind, int32_t dummy_player) {
  if (agent < 0 || agent > 1) return AZ_ERR_INVALID;
  GUARD_BEGIN
  std::unique_ptr<State> probe(make_state(e->d.game, e->d.flags));
  if (kind == AZ_INF_DUAL) e->inferers[agent] = std::make_shared<DualInferer>(*e->nets[agent]);
  else if (kind == AZ_INF_DUMMY) e->inferers[agent] = std::make_shared<DummyInferer>(probe->ActionSpace(), dummy_player);
  else if (kind == AZ_INF_TABLE) { if (!dynamic_cast<TableInferer*>(e->inferers[agent].get())) e->inferers[agent] = std::make_shared<TableInferer>(); }
  else return AZ_ERR_INVALID;
  GUARD_END(e)
  return AZ_OK;
}
int az_agent_set_table(az_engine* e, int32_t agent, int32_t n_rows, int32_t row_len, const float* policy_rows,
                       const float* values) {
  if (agent < 0 || agent > 1) return AZ_ERR_INVALID;
  auto t = std::make_shared<TableInferer>();
  for (int r = 0; r < n_rows; r++) {
    t->rows.emplace_back(policy_rows + (size_t)r * row_len, policy_rows + (size_t)(r + 1) * row_len);
    t->values.push_back(values[r]);
  }
  e->inferers[agent] = t;
  return AZ_OK;
}
int az_infer(az_engine* e, int32_t agent, const float* planes, int32_t n, float* policy, float* value) {
  if (agent < 0 || agent > 1) return AZ_ERR_INVALID;
  DualInferer* di = dynamic_cast<DualInferer*>(e->inferers[agent].get());
  if (!di) { e->err = "agent has no dual inferer (call az_agent_set_inferer(AZ_INF_DUAL))"; return AZ_ERR_STATE; }
  GUARD_BEGIN
  dual_infer(di->net, planes, n, policy, value);
  GUARD_END(e)
  return AZ_OK;
}
int az_infer_tower(az_engine* e, int32_t agent, const float* planes, int32_t n, float* tower_out) {
  if (agent < 0 || agent > 1 || n < 0) return AZ_ERR_INVALID;
  DualInferer* di = dynamic_cast<DualInferer*>(e->inferers[agent].get());
  if (!di) { e->err = "agent has no dual inferer (call az_agent_set_inferer(AZ_INF_DUAL))"; return AZ_ERR_STATE; }
  GUARD_BEGIN
  std::vector<float> policy((size_t)n * di->net.conf.ActionSpace), value(n), tower;
  dual_infer(di->net, planes, n, policy.data(), value.data(), &tower);
  std::copy(tower.begin(), tower.end(), tower_out);
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

static void add_counters(Counters& a, const Counters& b) {
  a.sims += b.sims; a.null_results += b.null_results; a.evals += b.evals; a.select_children += b.select_children;
  a.select_levels += b.select_levels; a.created += b.created; a.backup_nodes += b.backup_nodes; a.searches += b.searches;
}
static void harvest(az_engine* e, Arena& a) {
  add_counters(e->base, a.A.mcts->cnt); a.A.mcts->cnt = Counters();
  if (a.B.mcts != a.A.mcts) { add_counters(e->base, a.B.mcts->cnt); a.B.mcts->cnt = Counters(); }
}

int az_arena_begin(az_engine* e, int32_t n_games, int32_t record) {
  if (n_games < 1 || n_games > e->d.n_games) { e->err = "n_games out of range"; return AZ_ERR_INVALID; }
  if (!e->inferers[0] || (!e->inferers[1] && !(e->d.flags & AZ_FLAG_SHARED_TREE))) { e->err = "agents have no inferer"; return AZ_ERR_STATE; }
  GUARD_BEGIN
  e->slots.clear(); e->records.clear();
  e->ext_valid[0] = e->ext_valid[1] = false;
  e->n_active_games = n_games; e->record = record != 0; e->in_play = true;
  for (int g = 0; g < n_games; g++) {
    std::unique_ptr<Arena> a(new Arena(make_state(e->d.game, e->d.flags), e->nets[0], e->nets[1], e->mc, e->d.encoder, e->d.seed));
    a->max_moves = e->d.game.max_moves;
    a->shared_tree = (e->d.flags & AZ_FLAG_SHARED_TREE) != 0;
    a->games = e->games_started++;
    a->newTrees();
    a->A.inferer = e->inferers[0];
    a->B.inferer = e->inferers[1] ? e->inferers[1] : e->inferers[0];
    a->playBegin(e->coin.intn(2), e->record);
    e->slots.push_back(std::move(a));
  }
  GUARD_END(e)
  return AZ_OK;
}
static int count_active(az_engine* e) { int n = 0; for (auto& s : e->slots) n += s->active ? 1 : 0; return n; }
int az_search_begin(az_engine* e) {
  if (!e->in_play) return AZ_ERR_STATE;
  GUARD_BEGIN for (auto& s : e->slots) if (s->active) s->searchBegin(); GUARD_END(e)
  return AZ_OK;
}
int az_search_run(az_engine* e, int32_t n) {
  if (!e->in_play) return AZ_ERR_STATE;
  GUARD_BEGIN for (auto& s : e->slots) if (s->active) s->searchRun(n); GUARD_END(e)
  return AZ_OK;
}
int az_search_end(az_engine* e) {
  if (!e->in_play) return AZ_ERR_STATE;
  GUARD_BEGIN for (auto& s : e->slots) if (s->active) { s->searchEnd(); harvest(e, *s); } GUARD_END(e)
  return AZ_OK;
}
int az_arena_step(az_engine* e, int32_t* n_active) {
  int rc;
  if ((rc = az_search_begin(e))) return rc;
  if ((rc = az_search_run(e, e->mc.Sims))) return rc;
  if ((rc = az_search_end(e))) return rc;
  if (n_active) *n_active = count_active(e);
  return AZ_OK;
}
int az_arena_finish(az_engine* e) {
  if (!e->in_play) return AZ_ERR_STATE;
  GUARD_BEGIN
  for (auto& s : e->slots) {
    harvest(e, *s);
    std::vector<Example> ex = s->playFinish();
    e->examples.insert(e->examples.end(), ex.begin(), ex.end());
    e->records.push_back(s->records.back());
    e->wins[0] += s->A.Wins; e->loss[0] += s->A.Loss; e->draw[0] += s->A.Draw;
    e->wins[1] += s->B.Wins; e->loss[1] += s->B.Loss; e->draw[1] += s->B.Draw;
    s->A.resetStats(); s->B.resetStats();
  }
  e->in_play = false;
  GUARD_END(e)
  return AZ_OK;
}
int az_arena_play(az_engine* e, int32_t n_games, int32_t record) {
  int done = 0;
  std::vector<GameRecord> all;
  while (done < n_games) {
    int chunk = n_games - done < e->d.n_games ? n_games - done : e->d.n_games;
    int rc;
    if ((rc = az_arena_begin(e, chunk, record))) return rc;
    int na = count_active(e);
    while (na > 0) if ((rc = az_arena_step(e, &na))) return rc;
    if ((rc = az_arena_finish(e))) return rc;
    all.insert(all.end(), e->records.begin(), e->records.end());
    done += chunk;
  }
  e->records = all;
  return AZ_OK;
}

int az_search(az_engine* e, int32_t agent, const az_state* st, int32_t player, int32_t* best, float* child_visits) {
  if (agent < 0 || agent > 1 || !st || !st->board || st->n_hist < 0 || (st->n_hist > 0 && !st->hist)) return AZ_ERR_INVALID;
  if (st->n_hist > 8 && !(e->d.game.kind == AZ_GAME_WQ && (e->d.flags & AZ_FLAG_WQ_COMPLETE))) return AZ_ERR_INVALID;
  if (e->in_play) { e->err = "az_search during a running arena"; return AZ_ERR_STATE; }
  if (!e->inferers[agent]) { e->err = "agent has no inferer"; return AZ_ERR_STATE; }
  GUARD_BEGIN
  const az_game_desc& g = e->d.game;
  const int cells = g.m * g.n;
  std::unique_ptr<State> state;
  if (g.kind == AZ_GAME_MNK) {
    MNK* t = new MNK(g.m, g.n, g.k);
    t->board.assign(st->board, st->board + cells);
    t->history.assign(st->move_number, PlayerMove{None, st->last_move}); t->histPtr = st->move_number; t->nextToMove = st->to_move;
    for (int i = 0; i < st->n_moves && i < st->move_number; i++)  // the tail of the history the caller knows
      t->history[st->move_number - 1 - i] = PlayerMove{(Player)st->moves[2 * (st->n_moves - 1 - i)], (Single)st->moves[2 * (st->n_moves - 1 - i) + 1]};
    state.reset(t);
  } else if (g.kind == AZ_GAME_C4) {
    C4* t = new C4(g.m, g.n, g.k);
    t->data.assign(st->board, st->board + cells); t->nextToMove = st->to_move; t->passCount = st->passes;
    if (st->last_move != PassMove || st->move_number > 0) { t->history.assign(1, PlayerMove{None, st->last_move}); t->histPtr = 1; }
    state.reset(t);
  } else {
    WQ* t = new WQ(g.m, 0, g.komi, g.zobrist_seed);
    t->complete = (e->d.flags & AZ_FLAG_WQ_COMPLETE) != 0;
    t->ko = t->complete ? st->ko : -1;
    t->board.data.assign(st->board, st->board + cells);
    for (int i = 0; i < cells; i++) if (st->board[i]) t->board.zupdate(PlayerMove{st->board[i], (Single)i});  // clean hash
    t->nextToMove = st->to_move; t->passes = st->passes; t->moveCount = st->move_number;
    t->history.assign(st->move_number, PlayerMove{None, st->last_move}); t->histPtr = st->move_number;
    for (int i = 0; i < st->n_hist; i++) {
      if (st->move_number - st->n_hist + i < 0) continue;  // Historical(h) = the board before move h
      auto hn = std::make_shared<WQ::HistNode>();
      hn->board.assign(st->hist + (size_t)i * cells, st->hist + (size_t)(i + 1) * cells);
      hn->prev = t->hist; hn->idx = st->move_number - st->n_hist + i;
      t->hist = hn;
    }
    state.reset(t);
  }
  // The agent's MCTS survives the call when the position continues the one it searched last (include/agogo_b200.h,
  // az_search): same admission rule as the engine's host side — then MCTS.Search's own updateRoot / newRootState
  // (search.go:424-500) does the re-rooting, findChild failures included.
  const int ti = (e->d.flags & AZ_FLAG_SHARED_TREE) ? 0 : agent;
  const int depth = st->move_number - e->ext_prev_mn[ti];
  bool reuse = g.kind == AZ_GAME_MNK && e->ext_valid[ti] && e->ext_agent[ti] && depth >= 0 &&
               (depth == 0 || (st->moves && st->n_moves >= depth)) && st->move_number < cells + 2;
  if (reuse) {
    std::vector<int32_t> tmp(st->board, st->board + cells);
    for (int i = 0; i < depth && reuse; i++) {
      const int mv = st->moves[2 * (st->n_moves - 1 - i) + 1];
      if (mv < 0 || mv >= cells) reuse = false; else tmp[mv] = None;
    }
    if (reuse) reuse = tmp == e->ext_prev_board[ti];
  }
  if (!reuse) {
    e->ext_valid[ti] = false;
    e->ext_agent[ti].reset(new Agent);
    e->ext_agent[ti]->mcts.reset(new MCTS(state.get(), e->mc, e->ext_agent[ti].get(), derive_seed(derive_seed(e->d.seed, 1), ti)));
  }
  Agent& ag = *e->ext_agent[ti];
  ag.NN = e->nets[agent]; ag.enc = e->d.encoder; ag.player = player; ag.inferer = e->inferers[agent];
  Single b = ag.Search(state.get());
  e->ext_valid[ti] = true; e->ext_prev_mn[ti] = st->move_number; e->ext_prev_board[ti].assign(st->board, st->board + cells);
  add_counters(e->base, ag.mcts->cnt); ag.mcts->cnt = Counters();
  if (best) *best = b;
  if (child_visits) {
    int A = state->ActionSpace();
    for (int i = 0; i <= A; i++) child_visits[i] = 0;
    const MCTS& t = *ag.mcts;
    if (t.root != nilNode)
      for (int kid : t.children[t.root]) {
        int mv = t.nodes[kid].move;
        if (mv == PassMove) child_visits[A] = (float)t.nodes[kid].visits;
        else if (mv >= 0 && mv < A) child_visits[mv] = (float)t.nodes[kid].visits;
      }
  }
  GUARD_END(e)
  return AZ_OK;
}

int az_agent_reset_tree(az_engine* e, int32_t agent) {
  if (agent < 0 || agent > 1) return AZ_ERR_INVALID;
  if (e->in_play) { e->err = "az_agent_reset_tree during a running arena"; return AZ_ERR_STATE; }
  e->ext_valid[(e->d.flags & AZ_FLAG_SHARED_TREE) ? 0 : agent] = false;
  return AZ_OK;
}

int az_game_record(const az_engine* e, int32_t game, int32_t* moves, int32_t cap, int32_t* n_moves, int32_t* winner,
                   int32_t* a_player, int32_t* n_examples) {
  const GameRecord* r = nullptr;
  if (!e->in_play) { if (game < 0 || game >= (int)e->records.size()) return AZ_ERR_INVALID; r = &e->records[game]; }
  else { if (game < 0 || game >= (int)e->slots.size()) return AZ_ERR_INVALID; r = &e->slots[game]->rec; }
  int n = (int)r->moves.size();
  if (n_moves) *n_moves = n;
  if (moves) for (int i = 0; i < n && i < cap; i++) moves[i] = r->moves[i];
  if (winner) *winner = e->in_play ? e->slots[game]->winner : r->winner;
  if (a_player) *a_player = r->a_player;
  if (n_examples) *n_examples = e->in_play ? (int)e->slots[game]->examples.size() : r->n_examples;
  return AZ_OK;
}
int az_game_state(const az_engine* e, int32_t game, int32_t* board, int32_t cap, int32_t* to_move, int32_t* move_number,
                  int32_t* passes, int32_t* ended, int32_t* winner) {
  if (game < 0 || game >= (int)e->slots.size()) return AZ_ERR_INVALID;
  const State* s = e->slots[game]->game;
  const std::vector<int32_t>& b = s->Board();
  if (board) for (int i = 0; i < (int)b.size() && i < cap; i++) board[i] = b[i];
  if (to_move) *to_move = s->ToMove();
  if (move_number) *move_number = s->MoveNumber();
  if (passes) *passes = s->Passes();
  // ended/winner: what Arena.Play's loop condition last saw (arena.go:96)
  if (ended) *ended = e->slots[game]->lastEnded;
  if (winner) *winner = e->slots[game]->winner;
  return AZ_OK;
}
int az_examples_count(const az_engine* e, int64_t* n) { *n = (int64_t)e->examples.size(); return AZ_OK; }
int az_examples_read(const az_engine* e, int64_t start, int64_t n, float* boards, float* policies, float* values) {
  if (start < 0 || start + n > (int64_t)e->examples.size()) return AZ_ERR_INVALID;
  for (int64_t i = 0; i < n; i++) {
    const Example& ex = e->examples[start + i];
    if (boards) memcpy(boards + i * ex.Board.size(), ex.Board.data(), ex.Board.size() * 4);
    if (policies) memcpy(policies + i * ex.Policy.size(), ex.Policy.data(), ex.Policy.size() * 4);
    if (values) values[i] = ex.Value;
  }
  return AZ_OK;
}
int az_examples_clear(az_engine* e) { e->examples.clear(); return AZ_OK; }

int az_tree_dump(const az_engine* e, int32_t game, int32_t tree, int32_t* rows, int32_t cap_rows, int32_t* n_rows) {
  if (game < 0 || game >= (int)e->slots.size() || tree < 0 || tree > 1) return AZ_ERR_INVALID;
  const Arena& a = *e->slots[game];
  const MCTS* t = tree == 0 ? a.A.mcts.get() : a.B.mcts.get();
  std::vector<MCTS::DumpRow> out;
  if (t->root != nilNode) t->dump(t->root, 0, &out);
  *n_rows = (int32_t)out.size();
  for (int i = 0; i < (int)out.size() && i < cap_rows; i++) {
    int32_t* r = rows + (size_t)i * 7;
    r[0] = out[i].depth; r[1] = out[i].move; r[2] = (int32_t)out[i].visits; r[3] = (int32_t)out[i].wbits;
    r[4] = (int32_t)out[i].pbits; r[5] = out[i].expanded; r[6] = out[i].nchildren;
  }
  return AZ_OK;
}

int az_rules_apply(az_engine* e, int32_t n, const int32_t* boards, const int32_t* players, const int32_t* moves,
                   int32_t* check, int32_t* applied, int32_t* out_boards, int32_t* taken) {
  const az_game_desc& g = e->d.game;
  int cells = g.m * g.n;
  for (int i = 0; i < n; i++) {
    const int32_t* b = boards + (size_t)i * cells;
    int32_t* ob = out_boards + (size_t)i * cells;
    PlayerMove pm{players[i], moves[i]};
    check[i] = 0; applied[i] = 0; taken[i] = 0;
    memcpy(ob, b, cells * 4);
    try {
      if (g.kind == AZ_GAME_MNK) {
        MNK s(g.m, g.n, g.k); s.board.assign(b, b + cells);
        check[i] = s.Check(pm); applied[i] = check[i];
        s.Apply(pm); memcpy(ob, s.board.data(), cells * 4);
      } else if (g.kind == AZ_GAME_C4) {
        C4 s(g.m, g.n, g.k); s.data.assign(b, b + cells);
        check[i] = s.Check(pm);
        applied[i] = s.boardApply(pm);
        memcpy(ob, s.data.data(), cells * 4);
      } else {
        WQ s(g.m, 0, g.komi, g.zobrist_seed); s.board.data.assign(b, b + cells);
        s.complete = (e->d.flags & AZ_FLAG_WQ_COMPLETE) != 0;
        if (pm.single == PassMove) { check[i] = 1; applied[i] = 1; continue; }  // COMPLETION: pass is a board no-op
        if (pm.player == Black || pm.player == White) check[i] = s.Check(pm);
        if (s.complete) {  // stateless: no ko point
          std::vector<int> captured;
          const bool ok = (pm.player == Black || pm.player == White) && pm.single >= 0 && pm.single < cells && s.completeCheck(pm, &captured, nullptr);
          if (ok) { s.board.data[pm.single] = pm.player; for (int st : captured) s.board.data[st] = None; }
          applied[i] = ok; taken[i] = ok ? (int32_t)captured.size() : 0;
          memcpy(ob, s.board.data.data(), cells * 4);
          continue;
        }
        uint8_t t = 0;
        applied[i] = s.board.Apply(pm, &t);
        taken[i] = t;
        memcpy(ob, s.board.data.data(), cells * 4);
      }
    } catch (const std::exception&) { /* a reference panic: leave check/applied = 0 */ }
  }
  return AZ_OK;
}
int az_rules_status(az_engine* e, int32_t n, const int32_t* boards, const int32_t* passes, int32_t* ended,
                    int32_t* winner, float* score_black, float* score_white) {
  const az_game_desc& g = e->d.game;
  int cells = g.m * g.n;
  for (int i = 0; i < n; i++) {
    const int32_t* b = boards + (size_t)i * cells;
    std::unique_ptr<State> s;
    if (g.kind == AZ_GAME_MNK) { MNK* t = new MNK(g.m, g.n, g.k); t->board.assign(b, b + cells); s.reset(t); }
    else if (g.kind == AZ_GAME_C4) { C4* t = new C4(g.m, g.n, g.k); t->data.assign(b, b + cells); t->passCount = passes ? passes[i] : 0; s.reset(t); }
    else { WQ* t = new WQ(g.m, 0, g.komi, g.zobrist_seed); t->complete = (e->d.flags & AZ_FLAG_WQ_COMPLETE) != 0; t->board.data.assign(b, b + cells); t->passes = passes ? passes[i] : 0; s.reset(t); }
    Player w = None;
    ended[i] = s->Ended(&w);
    winner[i] = w;
    score_black[i] = s->Score(Black);
    score_white[i] = s->Score(White);
  }
  return AZ_OK;
}

int az_train(az_engine* e, int32_t net, float* Xs, float* Pi, float* V, int32_t batches, int32_t iterations, float lr,
             uint64_t shuffle_seed, float* costs_out) {
  if (net < 0 || net > 1) return AZ_ERR_INVALID;
  GUARD_BEGIN
  const DualConfig& c = e->dc;
  size_t rows = (size_t)batches * c.BatchSize;
  std::vector<float> x(Xs, Xs + rows * c.Features * c.Height * c.Width), p(Pi, Pi + rows * c.ActionSpace), v(V, V + rows);
  Rng r(shuffle_seed);
  std::vector<float> costs;
  dual_train(*e->nets[net], x, p, v, batches, iterations, lr, &r, &costs);
  memcpy(Xs, x.data(), x.size() * 4); memcpy(Pi, p.data(), p.size() * 4); memcpy(V, v.data(), v.size() * 4);
  if (costs_out) memcpy(costs_out, costs.data(), costs.size() * 4);
  GUARD_END(e)
  return AZ_OK;
}

int az_train_grads(az_engine* e, int32_t net, const float* X, const float* Pi, const float* V, float* grads_out,
                   float* cost_out) {
  if (net < 0 || net > 1) return AZ_ERR_INVALID;
  GUARD_BEGIN
  std::vector<float> g;
  float c = dual_train_step(*e->nets[net], X, Pi, V, 0.0f, &g);
  if (grads_out) memcpy(grads_out, g.data(), g.size() * 4);
  if (cost_out) *cost_out = c;
  GUARD_END(e)
  return AZ_OK;
}
int az_train_apply(az_engine* e, int32_t net, const float* grads, float lr) {
  if (net < 0 || net > 1) return AZ_ERR_INVALID;
  std::vector<float>& p = e->nets[net]->params;
  for (size_t i = 0; i < p.size(); i++) p[i] = p[i] - lr * grads[i];  // VanillaSolver (meta.go:20,39)
  return AZ_OK;
}

int az_comm_unique_id(uint8_t id[128]) { memset(id, 0, 128); return AZ_ERR_UNSUPPORTED; }
int az_comm_init(az_engine*, int32_t, int32_t, const uint8_t*) { return AZ_ERR_UNSUPPORTED; }

int az_comm_bench(az_engine*, int32_t, int32_t, double*, double*) { return AZ_ERR_UNSUPPORTED; }
int az_profile(az_engine*, int32_t, double out[8]) { if (out) for (int i = 0; i < 8; i++) out[i] = 0; return AZ_OK; }

int az_counters_get(const az_engine* e, az_counters* out) {
  memset(out, 0, sizeof *out);
  Counters c = e->base;
  for (auto& s : e->slots) { add_counters(c, s->A.mcts->cnt); if (s->B.mcts != s->A.mcts) add_counters(c, s->B.mcts->cnt); }
  out->searches = c.searches; out->sims = c.sims; out->null_results = c.null_results; out->evals = c.evals;
  out->select_children = c.select_children; out->select_levels = c.select_levels; out->created = c.created;
  out->backup_nodes = c.backup_nodes;
  return AZ_OK;
}
int az_counters_reset(az_engine* e) {
  e->base = Counters();
  for (auto& s : e->slots) { s->A.mcts->cnt = Counters(); s->B.mcts->cnt = Counters(); }
  return AZ_OK;
}

// Oracle-only extra: OpenMP thread count of the conv loops (bench.py picks the fastest setting on the box).
int azo_set_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
  return omp_get_max_threads();
#else
  return 1;
#endif
}

// Oracle-only extra: the reference's own AZ.Learn loop (agogo.go:100-172) run natively, used to
// check the host-side Learn composition.  out_log rows: 11 floats per epoch.
int azo_learn(const az_engine_desc* desc, double update_threshold, int32_t max_examples, int32_t iters, int32_t episodes,
              int32_t nniters, int32_t arena_games, float* out_log, float* out_final_params_a) {
  az_engine* e = nullptr;
  int rc = az_engine_create(desc, &e);
  if (rc) return rc;
  try {
    AZConfig c; c.nn = e->dc; c.mcts = e->mc; c.UpdateThreshold = update_threshold; c.MaxExamples = max_examples; c.enc = desc->encoder;
    AZ az(make_state(desc->game, desc->flags), c, desc->seed);
    az.arena->max_moves = desc->game.max_moves;
    az.Learn(iters, episodes, nniters, arena_games);
    for (size_t i = 0; i < az.log.size(); i++) {
      const EpochLog& l = az.log[i];
      float* o = out_log + i * 11;
      o[0] = l.a_wins; o[1] = l.a_loss; o[2] = l.a_draw; o[3] = l.b_wins; o[4] = l.b_loss; o[5] = l.b_draw;
      o[6] = (float)l.n_examples; o[7] = (float)l.batches; o[8] = (float)l.promoted; o[9] = l.first_cost; o[10] = l.last_cost;
    }
    if (out_final_params_a) memcpy(out_final_params_a, az.arena->A.NN->params.data(), az.arena->A.NN->params.size() * 4);
  } catch (const std::exception& ex) {
    g_create_error = ex.what();
    az_engine_destroy(e);
    return AZ_ERR_PANIC;
  }
  az_engine_destroy(e);
  return AZ_OK;
}

}  // extern "C"
