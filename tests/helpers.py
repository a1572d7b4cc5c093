"""Checks shared by the oracle tests (CPU, -m "not gpu") and the engine parity tests (-m gpu):
every function takes a bound library (agogo_b200._capi.Lib), so the same golden vectors pin the
oracle and then the CUDA engine."""
import numpy as np

from agogo_b200 import _capi as K
from tests.golden import rules_golden as G


def tiny_nn(m, n, A1, k=3, layers=1, fc=4, batch=4, features=2):
    return dict(k=k, shared_layers=layers, fc=fc, batch_size=batch, features=features, action_space=A1)


def rules_engine(lib, kind, m, n, k=0, komi=0.0):
    cells = m * n
    A = n if kind == K.GAME_C4 else cells
    d = K.make_desc(kind, m, n, k, komi=komi, sims=1, nn=tiny_nn(m, n, A + 1, features=2),
                    encoder=K.ENC_TWO_PLANE, n_games=1)
    return lib.create(d)


def check_mnk_golden(lib):
    for case in G.MNK:
        e = rules_engine(lib, K.GAME_MNK, case["m"], case["n"], case["k"])
        ended, winner, sb, sw = e.rules_status(np.array(case["board"], np.int32))
        if "is_winner" in case:  # isWinner(p) <=> Score(p) == 1 (mnk.go:142-150)
            score = sb[0] if case["is_winner"] == G.X else sw[0]
            assert score == 1.0, case
        if "ended" in case:
            assert ended[0] == case["ended"], case
        if "winner" in case:
            assert winner[0] == case["winner"], case
        e.close()


def check_c4_golden(lib):
    e = rules_engine(lib, K.GAME_C4, 6, 7, 4)
    boards = np.array([c["board"] for c in G.C4], np.int32)
    ended, winner, _, _ = e.rules_status(boards)
    for i, c in enumerate(G.C4):
        assert ended[i] == c["ended"], (i, c)
        assert winner[i] == c["winner"], (i, c)
    # gravity + full column + pass legality (c4.go:47-70)
    b = np.zeros((3, 42), np.int32)
    b[1, [0, 7, 14, 21, 28, 35]] = [1, 2, 1, 2, 1, 2]  # column 0 full
    check, applied, out, _ = e.rules_apply(b, [1, 1, 2], [3, 0, K.PASS])
    assert list(check) == [1, 0, 1] and list(applied) == [1, 0, 1]
    assert out[0, 35 + 3] == 1 and out[0].sum() == 1
    assert (out[1] == b[1]).all() and (out[2] == b[2]).all()
    e.close()


def check_wq_golden(lib):
    for i, c in enumerate(G.WQ):
        e = rules_engine(lib, K.GAME_WQ, c["size"], c["size"], 0)
        check, applied, out, taken = e.rules_apply(np.array(c["board"], np.int32), [c["player"]], [c["move"]])
        if c["err"]:
            assert applied[0] == 0, (i, c)
            assert (out[0] == np.array(c["board"])).all()
            if c["player"] != G.Z:
                assert check[0] == 0, (i, c)  # Game.Check also rejects (suicide / off-board)
        else:
            assert applied[0] == 1 and check[0] == 1, (i, c)
            assert taken[0] == c["taken"], (i, c)
            assert (out[0] == np.array(c["board2"])).all(), (i, c)
            _, _, sb, sw = e.rules_status(out[0])
            assert sw[0] == c["white"] and sb[0] == c["black"], (i, c, sb, sw)
        e.close()


def ttt_example_engine(lib, sims, n_games=1):
    """mcts/example_test.go:74-156: one MCTS searched by both colours, scripted dummyNN."""
    d = K.make_desc(K.GAME_MNK, 3, 3, 3, sims=sims, nn=tiny_nn(3, 3, 10), n_games=n_games,
                    flags=K.FLAG_SHARED_TREE, seed=7)
    e = lib.create(d)
    rows = np.zeros((10, 10), np.float32)
    vals = np.zeros(10, np.float32)
    for mn, (hot, p, v) in enumerate(G.TTT_DUMMY_NN):
        rows[mn, hot] = p
        vals[mn] = v
    e.set_inferer(0, K.INF_TABLE)
    e.set_table(0, rows, vals)
    return e


def check_ttt_kat(lib, sims):
    e = ttt_example_engine(lib, sims)
    e.arena_begin(1, False)
    n = 1
    while n:
        n = e.arena_step()
    rec = e.game_record(0)
    e.arena_finish()
    assert list(rec["moves"]) == G.TTT_EXPECTED_MOVES, (sims, rec)
    assert rec["winner"] == G.TTT_EXPECTED_WINNER
    e.close()


def play_and_collect(e, n_games, record=True, dump_trees=True, max_plies=10000):
    """Run begin/step*/finish; returns per-ply tree dumps (both trees of every game), records,
    examples, stats — everything parity compares."""
    e.examples(clear=True)
    e.arena_begin(n_games, record)
    shared = bool(e.desc.flags & K.FLAG_SHARED_TREE)
    dumps = []
    n, ply = n_games, 0
    while n and ply < max_plies:
        n = e.arena_step()
        if dump_trees:
            dumps.append([[e.tree_dump(g, t) for t in ((0,) if shared else (0, 1))] for g in range(n_games)])
        ply += 1
    states = [e.game_state(g) for g in range(n_games)]
    e.arena_finish()
    recs = [e.game_record(g) for g in range(n_games)]
    ex = e.examples(clear=True)
    stats = (e.stats(0), e.stats(1))
    return dict(dumps=dumps, records=recs, examples=ex, stats=stats, states=states, counters=e.counters())


def tree_children(rows):
    """Parent row of every row of a preorder tree dump (-1 for the root) and the children rows of every row, in list
    order: the children of row i are the next rows at depth + 1 until the depth drops back."""
    depth = rows[:, 0]
    parent = np.full(len(rows), -1, np.int64)
    kids = {}
    stack = []
    for i, d in enumerate(depth):
        while stack and depth[stack[-1]] >= d:
            stack.pop()
        if stack:
            parent[i] = stack[-1]
            kids.setdefault(stack[-1], []).append(i)
        stack.append(i)
    return parent, kids


def assert_same_run(a, b, what="", float_ulps=0):
    """float_ulps=0: every tree field bit-identical.  float_ulps>0 (network-in-the-loop runs only):
    structure, moves and visit counts identical, W and P within that many fp32 ulps — the engine's
    softmax/tanh use CUDA's expf/tanhf, the oracle glibc's, which differ in the last bit."""
    assert len(a["records"]) == len(b["records"])
    for g, (ra, rb) in enumerate(zip(a["records"], b["records"])):
        assert list(ra["moves"]) == list(rb["moves"]), (what, "moves", g, ra, rb)
        assert (ra["winner"], ra["a_player"], ra["n_examples"]) == (rb["winner"], rb["a_player"], rb["n_examples"]), (what, g, ra, rb)
    assert len(a["dumps"]) == len(b["dumps"]), (what, "plies")
    for ply, (da, db) in enumerate(zip(a["dumps"], b["dumps"])):
        for g, (ga, gb) in enumerate(zip(da, db)):
            for t, (ta, tb) in enumerate(zip(ga, gb)):
                assert ta.shape == tb.shape, (what, "tree size", ply, g, t, ta.shape, tb.shape)
                same = (ta == tb)
                if float_ulps:
                    for col in (3, 4):
                        fa, fb = ta[:, col].copy().view(np.float32), tb[:, col].copy().view(np.float32)
                        same[:, col] = np.abs(fa - fb) <= np.maximum(float_ulps * np.spacing(np.maximum(np.abs(fa), np.abs(fb))), 1e-5)
                if not same.all():
                    bad = np.argwhere((~same).any(axis=1))[0][0]
                    raise AssertionError("%s tree mismatch ply %d game %d tree %d row %d: %s vs %s" %
                                         (what, ply, g, t, bad, ta[bad], tb[bad]))
    for xa, xb in zip(a["examples"], b["examples"]):
        assert xa.shape == xb.shape, (what, "examples shape", xa.shape, xb.shape)
        assert (xa.view(np.uint32) == xb.view(np.uint32)).all(), (what, "examples bits")
    assert a["stats"] == b["stats"], (what, a["stats"], b["stats"])
    for k in ("searches", "sims", "null_results", "evals", "select_children", "select_levels", "created", "backup_nodes"):
        assert a["counters"][k] == b["counters"][k], (what, k, a["counters"], b["counters"])


def tame_gammas(engines, net, seed, target=0.9):
    """Random-init `net` identically in all engines, then rescale every BatchNorm scale tensor so that
    gamma/sqrt(eps) has std `target`.  With the reference's init (GlorotN over the full [B,C,H,W]
    shape) and its test-mode BN (x/sqrt(eps), see DESIGN.md) the per-layer gain is
    316*sqrt(2/((B+C)*H*W)), which only stays O(1) for the large configs; tiny test nets would
    overflow to inf/NaN in oracle and engine alike, which pins nothing."""
    e0 = engines[0]
    e0.net_init(net, seed)
    p = e0.net_get(net)
    nt, _ = e0.param_count()
    for i in range(nt):
        name, shape, off, size = e0.param_desc(i)
        if name.endswith("_γ"):
            g = p[off:off + size]
            g *= np.float32(target * np.sqrt(1e-5) / max(float(g.std()), 1e-12))
    for e in engines:
        e.net_set(net, p)
    return p


def check_workers_golden(lib):
    """tests/golden/workers_search.npz (tools/make_workers_golden.py): trees after the first Search and move records of
    games searched with mcts.Config workers > 1 under the fixed schedule."""
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tools"))
    import make_workers_golden as M
    gold = np.load(os.path.join(root, "tests", "golden", "workers_search.npz"))
    for name, desc, table, values in M.cases():
        trees, moves = M.run(lib, desc, table, values)
        for i, t in enumerate(trees):
            g = gold["%s_tree%d" % (name, i)]
            assert t.shape == g.shape and (t == g).all(), (name, "tree", i)
        for i, m in enumerate(moves):
            assert list(m) == list(gold["%s_moves%d" % (name, i)]), (name, "moves", i)
