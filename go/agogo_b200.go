// Package b200 is the cgo shim that puts the H100 engine (include/agogo_b200.h) under gorgonia/agogo's
// Go API.  UNCOMPILED in this repository's image (no Go toolchain); kept as the binding a maintainer
// would add next to agent.go / arena.go / agogo.go.  No Go pointer is retained by C after a call, and no Go-allocated
// struct containing Go pointers is passed to C (az_state's arrays are C.malloc copies).  backend_b200.go puts the
// reference's own method signatures — (*Agent).Search, (*Arena).Play, (*AZ).Learn, Save, Load — on top of this package.
package b200

/*
#cgo CFLAGS: -I${SRCDIR}/../include
#cgo LDFLAGS: -L${SRCDIR}/../agogo_b200 -lagogo_b200 -Wl,-rpath,${SRCDIR}/../agogo_b200
#include <stdlib.h>
#include "agogo_b200.h"
*/
import "C"

import (
	"errors"
	"unsafe"

	dual "github.com/gorgonia/agogo/dualnet"
	"github.com/gorgonia/agogo/game"
	"github.com/gorgonia/agogo/mcts"
)

// Engine owns the device state behind one agogo.AZ (two agents, two nets, n concurrent Arena games).
type Engine struct{ h *C.az_engine }

// Desc mirrors az_engine_desc; NN and MCTS are the reference's own config structs (source compatible).
type Desc struct {
	Kind, M, N, K int
	Komi          float32
	MaxMoves      int
	NN            dual.Config
	MCTS          mcts.Config
	Sims          int
	Workers       int // concurrent pipeline calls per tree (0/1 = canonical single worker)
	Encoder       int
	Games, Device int
	Seed          uint64
}

func check(e *Engine, rc C.int) error {
	if rc == C.AZ_OK {
		return nil
	}
	var h *C.az_engine
	if e != nil {
		h = e.h
	}
	msg := C.GoString(C.az_last_error(h))
	if rc == C.AZ_ERR_PANIC { // conditions on which the reference itself panics (node.go:232, agent.go:70)
		panic(msg)
	}
	return errors.New(msg)
}

// New replaces agogo.New (agogo.go:41-73): panics on invalid configs exactly like the reference.
func New(d Desc) *Engine {
	var cd C.az_engine_desc
	cd.game.kind, cd.game.m, cd.game.n, cd.game.k = C.int32_t(d.Kind), C.int32_t(d.M), C.int32_t(d.N), C.int32_t(d.K)
	cd.game.komi, cd.game.max_moves = C.float(d.Komi), C.int32_t(d.MaxMoves)
	m := d.MCTS
	cd.mcts.puct, cd.mcts.timeout_ns = C.float(m.PUCT), C.int64_t(m.Timeout)
	cd.mcts.m, cd.mcts.n, cd.mcts.random_count, cd.mcts.budget = C.int32_t(m.M), C.int32_t(m.N), C.int32_t(m.RandomCount), C.int32_t(m.Budget)
	cd.mcts.random_min_visits, cd.mcts.random_temperature = C.uint32_t(m.RandomMinVisits), C.float(m.RandomTemperature)
	if m.DumbPass {
		cd.mcts.dumb_pass = 1
	}
	cd.mcts.resign_percentage, cd.mcts.pass_preference, cd.mcts.sims = C.float(m.ResignPercentage), C.int32_t(m.PassPreference), C.int32_t(d.Sims)
	cd.mcts.workers = C.int32_t(d.Workers)
	n := d.NN
	cd.nn.k, cd.nn.shared_layers, cd.nn.fc, cd.nn.l2 = C.int32_t(n.K), C.int32_t(n.SharedLayers), C.int32_t(n.FC), C.double(n.L2)
	cd.nn.batch_size, cd.nn.width, cd.nn.height, cd.nn.features = C.int32_t(n.BatchSize), C.int32_t(n.Width), C.int32_t(n.Height), C.int32_t(n.Features)
	cd.nn.action_space = C.int32_t(n.ActionSpace)
	cd.encoder, cd.n_games, cd.device, cd.seed = C.int32_t(d.Encoder), C.int32_t(d.Games), C.int32_t(d.Device), C.uint64_t(d.Seed)
	e := &Engine{}
	if rc := C.az_engine_create(&cd, &e.h); rc != C.AZ_OK {
		panic(C.GoString(C.az_last_error(nil))) // agogo.go:42-47
	}
	return e
}

func (e *Engine) Close() { C.az_engine_destroy(e.h); e.h = nil }

// SetParams / Params move a dual.Dual's Model() tensors (dual.go:134-142 order) as one flat []float32;
// the Go *dual.Dual stays the checkpoint container, so AZ.Save/Load (agogo.go:175-209) keep working.
func (e *Engine) SetParams(net int, flat []float32) error {
	return check(e, C.az_net_set_params(e.h, C.int32_t(net), (*C.float)(unsafe.Pointer(&flat[0])), C.uint64_t(len(flat))))
}
func (e *Engine) Params(net int, flat []float32) error {
	return check(e, C.az_net_get_params(e.h, C.int32_t(net), (*C.float)(unsafe.Pointer(&flat[0])), C.uint64_t(len(flat))))
}

// SwitchToInference replaces Agent.SwitchToInference (agent.go:42-57); UseDummy replaces Agent.useDummy.
func (e *Engine) SwitchToInference(agent int) error {
	return check(e, C.az_agent_set_inferer(e.h, C.int32_t(agent), C.AZ_INF_DUAL, 0))
}
func (e *Engine) UseDummy(agent int, p game.Player) error {
	return check(e, C.az_agent_set_inferer(e.h, C.int32_t(agent), C.AZ_INF_DUMMY, C.int32_t(p)))
}

// Infer replaces Inferer.Infer (datatypes.go:51-55, meta.go:168-190), batched.
func (e *Engine) Infer(agent int, planes []float32, n int, policy, value []float32) error {
	return check(e, C.az_infer(e.h, C.int32_t(agent), (*C.float)(unsafe.Pointer(&planes[0])), C.int32_t(n),
		(*C.float)(unsafe.Pointer(&policy[0])), (*C.float)(unsafe.Pointer(&value[0]))))
}

// Play replaces a loop of Arena.Play(record, nil, nil) + game.Reset() (agogo.go:110-114, 144-148):
// nGames games run concurrently on the device; examples come back in game order.
func (e *Engine) Play(nGames int, record bool) error {
	r := C.int32_t(0)
	if record {
		r = 1
	}
	return check(e, C.az_arena_play(e.h, C.int32_t(nGames), r))
}

// Examples drains the recorded examples into agogo.Example-shaped slices (datatypes.go:38-42).
func (e *Engine) Examples(boardLen, policyLen int) (boards, policies, values []float32, err error) {
	var n C.int64_t
	if err = check(e, C.az_examples_count(e.h, &n)); err != nil || n == 0 {
		return
	}
	boards, policies, values = make([]float32, int(n)*boardLen), make([]float32, int(n)*policyLen), make([]float32, int(n))
	err = check(e, C.az_examples_read(e.h, 0, n, (*C.float)(unsafe.Pointer(&boards[0])), (*C.float)(unsafe.Pointer(&policies[0])),
		(*C.float)(unsafe.Pointer(&values[0]))))
	C.az_examples_clear(e.h)
	return
}

// Stats replaces reading Agent.Wins/Loss/Draw (agent.go:21-24).
func (e *Engine) Stats(agent int) (wins, loss, draw float32) {
	var w, l, d C.float
	C.az_agent_stats(e.h, C.int32_t(agent), &w, &l, &d)
	return float32(w), float32(l), float32(d)
}

// Train replaces dual.Train (meta.go:16-54).
func (e *Engine) Train(net int, Xs, Pi, V []float32, batches, iterations int, seed uint64) error {
	return check(e, C.az_train(e.h, C.int32_t(net), (*C.float)(unsafe.Pointer(&Xs[0])), (*C.float)(unsafe.Pointer(&Pi[0])),
		(*C.float)(unsafe.Pointer(&V[0])), C.int32_t(batches), C.int32_t(iterations), 0.1, C.uint64_t(seed), nil))
}

// InitNet replaces dual.New + Init (dual.go:33-48) and Arena.newB (arena.go:205-224): fresh random weights in `net`.
func (e *Engine) InitNet(net int, seed uint64) error {
	return check(e, C.az_net_init(e.h, C.int32_t(net), C.uint64_t(seed)))
}

// CopyNet replaces `A.NN = B.NN` on promotion (agogo.go:161).
func (e *Engine) CopyNet(dst, src int) error {
	return check(e, C.az_net_copy(e.h, C.int32_t(dst), C.int32_t(src)))
}

// ResetStats replaces Agent.resetStats (agent.go:115-121).
func (e *Engine) ResetStats(agent int) error {
	return check(e, C.az_agent_reset_stats(e.h, C.int32_t(agent)))
}

// cInts copies a Go []int32 into C memory (the cgo pointer-passing rule forbids handing C a Go struct that holds Go
// pointers: az_state's board / hist / moves therefore point at C allocations for the duration of the call).
func cInts(v []int32) *C.int32_t {
	if len(v) == 0 {
		return nil
	}
	p := (*C.int32_t)(C.malloc(C.size_t(len(v)) * 4))
	copy(unsafe.Slice((*int32)(unsafe.Pointer(p)), len(v)), v)
	return p
}

// Search replaces Agent.Search (agent.go:77-80) on a caller-owned game.State (GTP / analysis): the position is
// marshalled into an az_state — board colours, side to move, move number, passes, last move, up to 8 historical boards
// for the 18-plane encoder and the tail of the move history (what UndoLastMove / Fwd walk) — and searched for
// mcts.Config sims iterations.  The agent's device tree survives the call and is re-rooted on the next position when
// that continues this one (updateRoot, search.go:424-500); ResetTree is MCTS.Reset.  `history` = the state's
// (player, move) list, oldest first (mnk: State keeps it; pass nil when unknown: every call then searches a fresh tree).
// Returns the chosen move and the visit counts of the root's children ([A] + pass).
func (e *Engine) Search(agent int, s game.State, player game.Player, actionSpace int, history []game.PlayerMove) (game.Single, []float32, error) {
	raw := s.Board()
	board := make([]int32, len(raw))
	for i, c := range raw {
		board[i] = int32(c)
	}
	nHist := s.MoveNumber()
	if nHist > 8 {
		nHist = 8
	}
	var hist []int32
	for i := s.MoveNumber() - nHist; i < s.MoveNumber(); i++ { // oldest first; Historical(i) = board before move i
		for _, c := range s.Historical(i) {
			hist = append(hist, int32(c))
		}
	}
	moves := make([]int32, 0, 2*len(history))
	for _, pm := range history {
		moves = append(moves, int32(pm.Player), int32(pm.Single))
	}
	var st C.az_state // holds C pointers only
	st.board = cInts(board)
	defer C.free(unsafe.Pointer(st.board))
	st.to_move, st.move_number, st.passes = C.int32_t(s.ToMove()), C.int32_t(s.MoveNumber()), C.int32_t(s.Passes())
	st.last_move = C.int32_t(s.LastMove().Single)
	if len(hist) == nHist*len(board) && nHist > 0 {
		st.n_hist, st.hist = C.int32_t(nHist), cInts(hist)
		defer C.free(unsafe.Pointer(st.hist))
	}
	if len(moves) > 0 {
		st.n_moves, st.moves = C.int32_t(len(history)), cInts(moves)
		defer C.free(unsafe.Pointer(st.moves))
	}
	st.ko = -1 // simple ko is a property of OUR complete-rules mode; a reference game.State has none
	var best C.int32_t
	visits := make([]float32, actionSpace+1)
	err := check(e, C.az_search(e.h, C.int32_t(agent), &st, C.int32_t(player), &best, (*C.float)(unsafe.Pointer(&visits[0]))))
	return game.Single(best), visits, err
}

// ResetTree replaces MCTS.Reset (tree.go:249-276) for the agent's external-search tree.
func (e *Engine) ResetTree(agent int) error { return check(e, C.az_agent_reset_tree(e.h, C.int32_t(agent))) }

// Begin / Step / Finish expose Arena.Play's loop (arena.go:80-179) ply by ply for n concurrent games, so that a Go
// Arena can run its OutputEncoder between moves; GameRecord returns the moves of one of them.
func (e *Engine) Begin(nGames int, record bool) error {
	r := C.int32_t(0)
	if record {
		r = 1
	}
	return check(e, C.az_arena_begin(e.h, C.int32_t(nGames), r))
}
func (e *Engine) Step() (active int, err error) {
	var n C.int32_t
	err = check(e, C.az_arena_step(e.h, &n))
	return int(n), err
}
func (e *Engine) Finish() error { return check(e, C.az_arena_finish(e.h)) }
func (e *Engine) GameRecord(g, maxMoves int) (moves []int32, winner, aPlayer game.Player, err error) {
	moves = make([]int32, maxMoves)
	var n, w, ap, ne C.int32_t
	err = check(e, C.az_game_record(e.h, C.int32_t(g), (*C.int32_t)(unsafe.Pointer(&moves[0])), C.int32_t(maxMoves), &n, &w, &ap, &ne))
	if int(n) < maxMoves {
		moves = moves[:int(n)]
	}
	return moves, game.Player(w), game.Player(ap), err
}

// CommInit joins the gradient all-reduce group of a multi-process Learn (one process per GPU): rank 0 obtains the id
// with UniqueID and hands it to the other ranks (any host-side channel).  After it, Train reduces gradients over NVLink.
func UniqueID() ([128]byte, error) {
	var id [128]byte
	rc := C.az_comm_unique_id((*C.uint8_t)(unsafe.Pointer(&id[0])))
	return id, check(nil, rc)
}
func (e *Engine) CommInit(id [128]byte, rank, world int) error {
	return check(e, C.az_comm_init(e.h, C.int32_t(rank), C.int32_t(world), (*C.uint8_t)(unsafe.Pointer(&id[0]))))
}
