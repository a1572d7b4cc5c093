// +build b200

// Drop-in bodies for the hot-path methods of package agogo on top of the H100 engine (package b200, agogo_b200.go).
// UNCOMPILED here (no Go toolchain in this image).  A maintainer adds this file to the root package and tags the
// reference's own bodies `// +build !b200`: agent.go (Search, SwitchToInference, useDummy, resetStats), arena.go (Play,
// newB), agogo.go (New, SelfPlay, Learn, Save, Load).  Every signature below is the reference's, so callers — cmd/*,
// the GTP front-end, user programs — compile unchanged; Config.Encoder must be one of the encoders the engine implements
// on device (the two-plane encoder of cmd/tictactoe, or WQEncoder) and is named by EngineEncoder.
package agogo

import (
	"encoding/gob"
	"os"

	dual "github.com/gorgonia/agogo/dualnet"
	"github.com/gorgonia/agogo/game"
	"github.com/gorgonia/agogo/mcts"
	b200 "github.com/gorgonia/agogo/b200"
	"github.com/pkg/errors"
	"gorgonia.org/tensor"
)

// engineOf is the one engine behind an AZ: agent 0 = A, agent 1 = B.  Set by New.
type b200State struct {
	eng         *b200.Engine
	games       int // concurrent device games (Config extension: B200Games, default 1024)
	seed        uint64
	boardLen    int
	actionSpace int
	history     []game.PlayerMove // of a.game, kept by Play / Search callers for tree reuse
}

var engines = map[*Arena]*b200State{}

func (a *Arena) b200() *b200State { return engines[a] }

// flat view of a *dual.Dual's Model() (dual.go:134-142 order): the engine's parameter layout
func modelToFlat(d *dual.Dual) []float32 {
	var out []float32
	for _, n := range d.Model() {
		out = append(out, n.Value().Data().([]float32)...)
	}
	return out
}
func flatToModel(flat []float32, d *dual.Dual) {
	off := 0
	for _, n := range d.Model() {
		dst := n.Value().Data().([]float32)
		copy(dst, flat[off:off+len(dst)])
		off += len(dst)
	}
}

// New replaces agogo.New (agogo.go:41-73): same panics, same fields; additionally creates the device engine and
// uploads both freshly initialised nets.
func New(g game.State, conf Config) *AZ {
	if !conf.NNConf.IsValid() {
		panic("NNConf is not valid. Unable to proceed")
	}
	if !conf.MCTSConf.IsValid() {
		panic("MCTSConf is not valid. Unable to proceed")
	}
	a := dual.New(conf.NNConf)
	b := dual.New(conf.NNConf)
	if err := a.Init(); err != nil {
		panic(err)
	}
	if err := b.Init(); err != nil {
		panic(err)
	}
	retVal := &AZ{
		Arena:           MakeArena(g, a, b, conf.MCTSConf, conf.Encoder, conf.Augmenter, conf.Name),
		nnConf:          conf.NNConf,
		mctsConf:        conf.MCTSConf,
		enc:             conf.Encoder,
		outEnc:          conf.OutputEncoder,
		aug:             conf.Augmenter,
		updateThreshold: float32(conf.UpdateThreshold),
		maxExamples:     conf.MaxExamples,
		Statistics:      makeStatistics(),
		useDummy:        true,
	}
	kind, m, n, k, komi := EngineGame(g) // mnk / c4 / wq and their parameters, from the concrete State type
	st := &b200State{games: 1024, seed: 1, boardLen: conf.NNConf.Features * conf.NNConf.Height * conf.NNConf.Width,
		actionSpace: g.ActionSpace()}
	st.eng = b200.New(b200.Desc{Kind: kind, M: m, N: n, K: k, Komi: komi, NN: conf.NNConf, MCTS: conf.MCTSConf,
		Sims: int(conf.MCTSConf.Budget), Encoder: EngineEncoder(conf.Encoder), Games: st.games, Seed: st.seed})
	engines[&retVal.Arena] = st
	must(st.eng.SetParams(0, modelToFlat(a)))
	must(st.eng.SetParams(1, modelToFlat(b)))
	return retVal
}

func must(err error) {
	if err != nil {
		panic(err)
	}
}

// Search replaces (*Agent).Search (agent.go:77-80).  The Agent knows its Arena through the engines table.
func (a *Agent) Search(g game.State) game.Single {
	ar, idx := arenaOf(a)
	st := ar.b200()
	best, _, err := st.eng.Search(idx, g, a.Player, st.actionSpace, st.history)
	if err != nil {
		panic(err) // agent.go:66-71: inference errors panic
	}
	return best
}

// SwitchToInference / useDummy / resetStats (agent.go:42-57, 105-121)
func (a *Agent) SwitchToInference(g game.State) error {
	ar, idx := arenaOf(a)
	must(ar.b200().eng.SetParams(idx, modelToFlat(a.NN)))
	return ar.b200().eng.SwitchToInference(idx)
}
func (a *Agent) useDummy(g game.State) {
	ar, idx := arenaOf(a)
	must(ar.b200().eng.UseDummy(idx, a.Player))
}
func (a *Agent) resetStats() {
	ar, idx := arenaOf(a)
	must(ar.b200().eng.ResetStats(idx))
	a.Wins, a.Loss, a.Draw = 0, 0, 0
}

// Play replaces (*Arena).Play (arena.go:80-179): ONE game on the device, stepped ply by ply so that the
// OutputEncoder sees the MetaState after every move exactly as arena.go:131-133 does; the Augmenter is applied to
// every kept example (arena.go:115-121).  Returns game.None like the reference (arena.go:178).
func (a *Arena) Play(record bool, enc OutputEncoder, aug Augmenter) (winner game.Player, examples []Example) {
	st := a.b200()
	must(st.eng.Begin(1, record))
	_, _, aPlayer, _ := st.eng.GameRecord(0, 1)
	a.A.Player, a.B.Player = aPlayer, opponent(aPlayer)
	a.currentPlayer = a.A
	if aPlayer != game.Player(game.Black) {
		a.currentPlayer = a.B
	}
	a.game.SetToMove(a.currentPlayer.Player)
	st.history = st.history[:0]
	for active := 1; active > 0; {
		var err error
		if active, err = st.eng.Step(); err != nil {
			panic(err)
		}
		moves, _, _, _ := st.eng.GameRecord(0, 2*len(a.game.Board())+4)
		pm := game.PlayerMove{Player: a.currentPlayer.Player, Single: game.Single(moves[len(moves)-1])}
		a.game = a.game.Apply(pm) // keep the Go-side MetaState in step with the device
		st.history = append(st.history, pm)
		a.switchPlayer()
		if enc != nil {
			enc.Encode(a)
		}
	}
	must(st.eng.Finish())
	boards, pols, vals, err := st.eng.Examples(st.boardLen, st.actionSpace+1)
	must(err)
	for i := range vals {
		ex := Example{Board: boards[i*st.boardLen : (i+1)*st.boardLen], Policy: pols[i*(st.actionSpace+1) : (i+1)*(st.actionSpace+1)], Value: vals[i]}
		if aug != nil {
			examples = append(examples, aug(ex)...)
		} else {
			examples = append(examples, ex)
		}
	}
	a.syncStats()
	return game.Player(game.None), examples
}

// PlayN is the batched form Learn uses: n games run concurrently on the device (n Arena.Play + game.Reset calls of
// agogo.go:110-114 / 144-148 in one call); examples come back in game order, Augmenter applied.
func (a *Arena) PlayN(n int, record bool, aug Augmenter) (examples []Example) {
	st := a.b200()
	must(st.eng.Play(n, record))
	boards, pols, vals, err := st.eng.Examples(st.boardLen, st.actionSpace+1)
	must(err)
	for i := range vals {
		ex := Example{Board: boards[i*st.boardLen : (i+1)*st.boardLen], Policy: pols[i*(st.actionSpace+1) : (i+1)*(st.actionSpace+1)], Value: vals[i]}
		if aug != nil {
			examples = append(examples, aug(ex)...)
		} else {
			examples = append(examples, ex)
		}
	}
	a.syncStats()
	return examples
}

func (a *Arena) syncStats() {
	st := a.b200()
	a.A.Wins, a.A.Loss, a.A.Draw = st.eng.Stats(0)
	a.B.Wins, a.B.Loss, a.B.Draw = st.eng.Stats(1)
}

// SelfPlay replaces (*AZ).SelfPlay (agogo.go:93-97).
func (a *AZ) SelfPlay() []Example {
	_, examples := a.Play(true, nil, a.aug)
	a.game.Reset()
	return examples
}

// Learn replaces (*AZ).Learn (agogo.go:100-172): same sequence, same promotion rule; self-play and arena games run
// as device batches, dual.Train on device (multi-GPU: one process per GPU, b200.CommInit before Learn).
func (a *AZ) Learn(iters, episodes, nniters, arenaGames int) error {
	st := a.b200()
	for a.epoch = 0; a.epoch < iters; a.epoch++ {
		a.setupSelfPlay(a.epoch)
		ex := a.PlayN(episodes, true, a.aug)
		if a.maxExamples > 0 && len(ex) > a.maxExamples {
			shuffleExamples(ex)
			ex = ex[:a.maxExamples]
		}
		Xs, Policies, Values, batches := a.prepareExamples(ex)
		if batches == 0 {
			return errors.New("batches is nil, probably too few examples regarding the batchsize")
		}
		if err := st.eng.Train(1, Xs.Data().([]float32), Policies.Data().([]float32), Values.Data().([]float32), batches, nniters,
			st.seed+uint64(a.epoch)); err != nil {
			return errors.WithMessage(err, "Train fail")
		}
		must(st.eng.SwitchToInference(1)) // a.B.SwitchToInference(a.game): the engine snapshots its own trained copy
		a.A.resetStats()
		a.B.resetStats()
		a.PlayN(arenaGames, false, nil)
		var killedA bool
		if a.B.Wins/(a.B.Wins+a.A.Wins) > a.updateThreshold { // NaN (0/0) never promotes, as in the reference
			must(st.eng.CopyNet(0, 1)) // a.A.NN = a.B.NN
			flat := make([]float32, len(modelToFlat(a.B.NN)))
			must(st.eng.Params(1, flat))
			flatToModel(flat, a.A.NN) // keep the Go-side container current for Save
			killedA = true
		}
		a.update(a.A)
		must(st.eng.InitNet(1, st.seed+1000+uint64(a.epoch))) // newB (arena.go:205-224): fresh random B every epoch
		_ = killedA
	}
	return nil
}

// Save / Load (agogo.go:175-209) keep the reference's gob container of a.A.NN; the engine only syncs the flat Model()
// payload in and out of the Go *dual.Dual.
func (a *AZ) Save(filename string) error {
	st := a.b200()
	flat := make([]float32, len(modelToFlat(a.A.NN)))
	if err := st.eng.Params(0, flat); err != nil {
		return err
	}
	flatToModel(flat, a.A.NN)
	f, err := os.OpenFile(filename, os.O_CREATE|os.O_TRUNC|os.O_WRONLY, 0544)
	if err != nil {
		return err
	}
	defer f.Close()
	return gob.NewEncoder(f).Encode(a.A.NN)
}

func (a *AZ) Load(filename string) error {
	f, err := os.Open(filename)
	if err != nil {
		return errors.WithStack(err)
	}
	defer f.Close()
	a.A.NN = dual.New(a.nnConf)
	a.B.NN = dual.New(a.nnConf)
	if err = gob.NewDecoder(f).Decode(a.A.NN); err != nil {
		return errors.WithStack(err)
	}
	f.Seek(0, 0)
	if err = gob.NewDecoder(f).Decode(a.B.NN); err != nil {
		return errors.WithStack(err)
	}
	st := a.b200()
	must(st.eng.SetParams(0, modelToFlat(a.A.NN)))
	must(st.eng.SetParams(1, modelToFlat(a.B.NN)))
	a.useDummy = false
	return nil
}

// ---- small helpers ---------------------------------------------------------------------------------------------------
func opponent(p game.Player) game.Player {
	if p == game.Player(game.Black) {
		return game.Player(game.White)
	}
	return game.Player(game.Black)
}

// arenaOf finds the Arena (and agent index) an Agent belongs to.
func arenaOf(a *Agent) (*Arena, int) {
	for ar := range engines {
		if ar.A == a {
			return ar, 0
		}
		if ar.B == a {
			return ar, 1
		}
	}
	panic("agent without an engine")
}

// EngineGame names the device rules for a concrete game.State (mnk.MNK, c4.Game, wq.Game) and their parameters.
// EngineEncoder names the device encoder for a GameEncoder (0: two-plane, 1: WQEncoder).  Both are a type switch over
// the reference's own types in the real package; kept as variables here so that programs can register others.
var EngineGame func(g game.State) (kind, m, n, k int, komi float32)
var EngineEncoder func(enc GameEncoder) int

var _ = tensor.Float32
var _ mcts.Config
