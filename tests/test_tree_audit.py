"""Every prior and value that self-play stores in its trees, checked against the network on that node's position.

The kernels are pinned one at a time elsewhere; this file checks how they combine inside the self-play wave: the leaf
planes written into slot agent * GS + slot0 + worker * active of the evaluation batch, the tower and heads run on the
batch count read from the device inside the replayed graph, and k_expand_backup's masking, normalisation, sort and
backup of policy[slot] / value[slot].  After every az_arena_step the tree of the agent that just moved is dumped, and:

  * its root position is rebuilt from the game record minus the last move (for az_search: the caller's state, earlier
    boards included), every expanded node's position by applying its path with the Python restatements of the rules
    (tests/pyref_mcts.py), with the search's own side-to-move bookkeeping (c4's Apply does not flip the player);
  * the encoder planes of every expanded node go through az_infer of a twin engine (same descriptor, same nets, so the
    same GS, tower kernels and heads block size) and k_expand_backup is restated in numpy float32: legal list = the
    node's children in index order with Pass last, Pass from pol[L-1], legalSum summed sequentially, correctly rounded
    division (uniform below 2^-149), stable descending sort;
  * priors bit for bit (order and every P bit; the root's children are re-sorted by bestMove, so there the prior of
    every move); leaf values bit for bit: W of a non-root expanded node whose children all have N = 1 is the sequential
    fp32 sum of k = N - 1 - sum(N_c - 1) copies of v' (v for Black to move, fl(1 - v) for White; k >= 2 where workers
    collided); internal nodes within the a-priori bound of sequential fp32 sums;
  * the twin's heads against the float64 heads on its own tower output, and az_infer bits independent of where a row
    sits in the batch (reversed, shifted by one slot, alone).

Every move is sampled from the root's visits, so the games diverge.  The test asserts that at least three quarters of
the audited games in neighbouring slots hold different positions.  It also asserts that exchanging those games'
outputs fails the audit, so the slot addressing is pinned, not only the per-sample arithmetic.  WQEncoder never encodes
the last two boards, so wq siblings are the same network input; an exchange of siblings' outputs is caught in the mnk
and c4 cases only.

On the CPU the oracle audits itself (it evaluates every sample with dual_infer, in search and in az_infer alike).  Each
of seven plausible faults restated in the auditor must make it fail in every case where it applies (fault_applies).
The CPU part takes about 5 s.

Measured on an H100 SXM (80 GB, 700 W): the eight GPU cases take 30 s in all (7.3 s the longest, wq13-k128-complete).
Every prior and every checked leaf value matched bit for bit.  Expanded nodes audited (leaf values checked;
neighbouring audited pairs holding different positions): c3-width 714 (650; 22 of 22), c3-width-workers 726 (504, 22
nodes with k >= 2; 22 of 22), c2 2150 (972; 48 of 48, 256 games moving at the first ply, 239 at the last),
c2-fp16 1162 (1088; 20 of 20), wq13-k128-complete 3200 (2273; 124 of 124), mnk13x9-k64 4800 (4530; 186 of 186),
c4-k16 5376 (4096; 246 of 252), external 66 (47).  The heads against float64 on up to 96 distinct rows per case: policy
at most 3.2e-7 relative, value 5.7e-8 absolute.
"""
import collections
import copy
import math

import numpy as np
import pytest

from agogo_b200 import _capi as K
from tests import helpers as H
from tests import pyref_dual as D
from tests import pyref_mcts as R
from tests.test_tc_layers import NUM_SMS, TOL_POLICY, TOL_VALUE, tower_layout

f32 = np.float32
TINY = np.finfo(np.float32).smallest_subnormal  # math32.SmallestNonzeroFloat32 = 2^-149
U = 2.0 ** -24
FAULTS = ("stale-history", "parent-position", "no-white-flip", "sibling-swap", "neighbour-slot", "pass-entry",
          "sorted-legalsum")


def fault_applies(fault, c):
    """Where a fault changes what the network sees or what the tree stores, so the audit must fail."""
    if fault == "stale-history":  # only WQEncoder has history planes
        return c.kind == K.GAME_WQ
    if fault == "sibling-swap":  # WQEncoder never encodes the last two boards: siblings are the same network input
        return c.kind != K.GAME_WQ
    if fault == "pass-entry":  # mnk has no Pass
        return c.kind != K.GAME_MNK
    return True

Case = collections.namedtuple("Case", "name kind m n win komi flags K layers fc games workers sims plies audit seed first "
                                      "pass_logit", defaults=(0, 0.0))
# audit: None = every game that moved; n = up to 2 * (4 + n / 2) games per agent and ply, in neighbouring-slot pairs
# (choose_games).  first: the first ply audited.  Every move is sampled from the root's visits (RandomCount = plies,
# temperature 1), so games diverge from the second ply on and neighbouring slots hold different positions; WQEncoder's
# planes are the boards before the last two moves, so the wq cases audit from the ply where those hold sampled stones.
# pass_logit: added to the nets' Pass logit (with PreferPass) so that games end by two passes at different plies and
# the evaluation batch shrinks.
CPU_CASES = [
    Case("ttt-k3", K.GAME_MNK, 3, 3, 3, 0.0, 0, 3, 1, 4, 6, 1, 12, 9, None, 3, 1),
    Case("c4-k16-shared-w4", K.GAME_C4, 6, 7, 4, 0.0, K.FLAG_SHARED_TREE, 16, 1, 8, 6, 4, 16, 8, None, 5, 2),
    Case("wq7-k4-w3", K.GAME_WQ, 7, 7, 0, 5.5, 0, 4, 1, 8, 6, 3, 16, 11, None, 7, 3),
    Case("wq5-k4-complete", K.GAME_WQ, 5, 5, 0, 5.5, K.FLAG_WQ_COMPLETE, 4, 1, 8, 6, 1, 24, 12, None, 9, 3),
]
GPU_CASES = [
    Case("c3-width", K.GAME_WQ, 19, 19, 0, 7.5, 0, 256, 2, 512, 1024, 1, 16, 6, 8, 11, 4),
    Case("c3-width-workers", K.GAME_WQ, 19, 19, 0, 7.5, 0, 256, 2, 512, -(-8 * NUM_SMS // 2) + 16, 2, 16, 6, 8, 13, 4),
    Case("c2", K.GAME_WQ, 9, 9, 0, 7.5, 0, 64, 6, 128, 256, 1, 32, 10, 8, 15, 4, 4.0),
    Case("c2-fp16", K.GAME_WQ, 9, 9, 0, 7.5, K.FLAG_FP16_TOWER, 64, 6, 128, 150, 2, 32, 6, 8, 17, 4),
    Case("wq13-k128-complete", K.GAME_WQ, 13, 13, 0, 7.5, K.FLAG_WQ_COMPLETE, 128, 2, 64, 64, 1, 24, 5, None, 19, 3),
    Case("mnk13x9-k64", K.GAME_MNK, 13, 9, 5, 0.0, 0, 64, 2, 64, 64, 1, 24, 4, None, 21, 1),
    Case("c4-k16", K.GAME_C4, 6, 7, 4, 0.0, K.FLAG_SHARED_TREE, 16, 2, 64, 64, 4, 32, 6, None, 23, 2),
]
# az_search on caller-owned 19x19 positions under the complete rules (the GTP front end's path), both agents
EXTERNAL = Case("external", K.GAME_WQ, 19, 19, 0, 7.5, K.FLAG_WQ_COMPLETE, 256, 2, 64, 1, 1, 32, 12, None, 25)


def action_space(c):
    return c.n if c.kind == K.GAME_C4 else c.m * c.n


def desc_of(c):
    feats = 18 if c.kind == K.GAME_WQ else 2
    d = K.make_desc(c.kind, c.m, c.n, c.win, komi=c.komi, sims=c.sims, n_games=c.games, seed=c.seed, flags=c.flags,
                    max_moves=c.plies, workers=c.workers,
                    pass_preference=K.PREFER_PASS if c.pass_logit else K.DONT_PREFER_PASS,
                    nn=dict(k=c.K, shared_layers=c.layers, fc=c.fc, batch_size=2, features=feats,
                            action_space=action_space(c) + 1))
    d.mcts.random_count, d.mcts.random_temperature = c.plies, 1.0
    return d


# ---------------------------------------------------------------------------------------------------------------------
# restated dispatch: which kernels a case runs (nn_fp32.cu heads_tiled, tower_tc.cu tc_tower_alloc)
def slot_count(c):
    return c.games * max(c.workers, 1)


def heads_block(gs):
    """k_heads_tiled<SB>: the most samples per block that still give every SM a block, from the slot capacity GS"""
    for sb in (8, 4, 2):
        if gs >= sb * NUM_SMS:
            return sb
    return 1


def uses_tensor_cores(c):
    return not (c.flags & K.FLAG_FP32_TOWER) and c.K in (64, 128, 256)


def tower_family(c):
    if not uses_tensor_cores(c):
        return "fp32 k_unit_f32"
    lay = tower_layout(c.m, c.n, c.K, c.layers)
    fp16 = bool(c.flags & K.FLAG_FP16_TOWER)
    if lay["small"]:
        return "k_smallnet_fp16" if fp16 else "k_net_small"
    conv = "k_conv3x3_tc fp16" if fp16 else ("k_conv3x3_m192" if c.K >= 128 else "k_conv3x3_tc")
    return "%s %s" % (conv, "per-sample" if lay["per_sample"] else "flat")


def heads_kernel(c, gs):
    return "k_heads_tiled<%d>" % heads_block(gs) if uses_tensor_cores(c) else "k_heads_f32"


# ---------------------------------------------------------------------------------------------------------------------
# positions
def new_game(c):
    if c.kind == K.GAME_MNK:
        return R.MNK(c.m, c.n, c.win)
    if c.kind == K.GAME_C4:
        return R.C4(c.m, c.n, c.win)
    return (R.WQComplete if c.flags & K.FLAG_WQ_COMPLETE else R.WQ)(c.m, c.komi)


def replay(c, moves):
    """The game after `moves`, Black moving first (Arena.Play gives Black to whichever agent starts)"""
    g = new_game(c)
    for i, mv in enumerate(moves):
        g = g.apply(R.BLACK if i % 2 == 0 else R.WHITE, int(mv))
    return g


def child_state(s, move):
    # the search applies the move for cur.next; mnk and wq then switch sides, c4 keeps the player (c4/game.go:55-72).
    # WQ.apply returns a new state; the others apply in place (and c4's Clone pads its history, so it is not used)
    return (s if isinstance(s, R.WQ) else copy.deepcopy(s)).apply(s.next, int(move))


def encode(c, s, stale=False):
    if c.kind != K.GAME_WQ:
        return R.encode_two_plane(s)
    if stale:  # fault: the history planes of one ply earlier
        s = s.clone()
        s.history, s.historical = s.history[:-1], s.historical[:-1]
    return R.encode_wq18(s)


# ---------------------------------------------------------------------------------------------------------------------
class Tree:
    """One dumped tree and the rebuilt position of each of its expanded nodes."""

    def __init__(self, rows, root, agent, ply, slot, label):
        self.rows, self.agent, self.ply, self.slot, self.label = rows, agent, ply, slot, label
        self.parent, self.kids = H.tree_children(rows)
        self.expanded = [i for i in range(len(rows)) if rows[i, 5]]
        self.states = {0: root}
        for i in self.expanded[1:]:  # preorder: a parent's state is built before its children's
            self.states[i] = child_state(self.states[self.parent[i]], rows[i, 1])
        self.idx = {}


class Run:
    """Trees of one case and the twin's outputs on their expanded nodes' planes."""

    def __init__(self, c, lib):
        self.c, self.lib = c, lib
        self.trees, self.planes = [], ([], [])
        self.slots = collections.Counter()
        self.active = []  # games that moved, per ply

    def add(self, tree):
        for i in tree.expanded:
            tree.idx[i] = len(self.planes[tree.agent])
            self.planes[tree.agent].append(encode(self.c, tree.states[i]))
        self.trees.append(tree)

    def partners(self):
        """Each audited tree's neighbour in the same wave: the tree one slot up, else one slot down (None if neither)"""
        at = {(t.ply, t.agent, t.slot): t for t in self.trees}
        return {id(t): at.get((t.ply, t.agent, t.slot + 1), at.get((t.ply, t.agent, t.slot - 1))) for t in self.trees}

    def distinct_neighbours(self):
        """Neighbouring audited trees whose root planes differ, and all such pairs"""
        partner = self.partners()
        pairs = [(t, partner[id(t)]) for t in self.trees if partner[id(t)] is not None and partner[id(t)].slot == t.slot + 1]
        diff = sum(bool((self.planes[t.agent][t.idx[0]] != self.planes[p.agent][p.idx[0]]).any()) for t, p in pairs)
        return diff, len(pairs)

    def evaluate(self, twin, stale=False):
        outs = []
        for a in (0, 1):  # one forward per agent: rows sit at slots 0.. of the twin's batch
            if stale:
                p = [encode(self.c, t.states[i], stale=True) for t in self.trees if t.agent == a for i in t.expanded]
            else:
                p = self.planes[a]
            outs.append(twin.infer(a, np.array(p, np.float32)) if p else None)
        return outs


def choose_games(moved, sb, n_pick):
    """Slots to audit among the games that moved (slot order per agent), in neighbouring pairs: the first and last slot
    of a heads block and across its boundary, the last (possibly partial) block, the last slot, and evenly spaced
    others."""
    cnt = len(moved)
    if n_pick is None or cnt <= n_pick:
        return list(range(cnt))
    anchors = {0, sb - 1, (cnt - 1) // sb * sb, cnt - 2} | set(np.linspace(0, cnt - 2, n_pick // 2).astype(int).tolist())
    return sorted({t for s in anchors if 0 <= s < cnt - 1 for t in (s, s + 1)})


def make_engines(lib, c):
    e, twin = lib.create(desc_of(c)), lib.create(desc_of(c))
    for a in (0, 1):
        p = H.tame_gammas([e, twin], a, 100 * c.seed + a)
        if c.pass_logit:
            off, size = next((off, size) for name, _, off, size in map(e.param_desc, range(e.param_count()[0]))
                             if name == "Policy_b")
            p[off + action_space(c):off + size:action_space(c) + 1] += f32(c.pass_logit)  # every row's Pass entry
            e.net_set(a, p)
            twin.net_set(a, p)
        e.set_inferer(a, K.INF_DUAL)
        twin.set_inferer(a, K.INF_DUAL)
    return e, twin


def collect_arena(lib, c):
    e, twin = make_engines(lib, c)
    run = Run(c, lib)
    shared = bool(c.flags & K.FLAG_SHARED_TREE)
    sb = heads_block(slot_count(c))
    e.arena_begin(c.games, False)
    for ply in range(c.plies):
        n_active = e.arena_step()
        recs = [e.game_record(g) for g in range(c.games)]
        moved = [g for g in range(c.games) if len(recs[g]["moves"]) == ply + 1]
        run.active.append(len(moved))
        by_agent = {0: [], 1: []}
        for g in moved:  # k_assign_slots: a game's slot is its rank among the active games of the agent to move
            first = 0 if recs[g]["a_player"] == R.BLACK else 1
            by_agent[0 if shared else first ^ (ply & 1)].append(g)
        for agent, games in by_agent.items():
            for slot in (choose_games(games, sb, c.audit) if ply >= c.first else []):
                g = games[slot]
                moves = recs[g]["moves"]
                root = replay(c, moves[:-1])
                root.next = R.BLACK if ply % 2 == 0 else R.WHITE
                st = e.game_state(g)
                after = child_state(root, moves[-1])
                assert list(after.board) == list(st["board"]), (c.name, "rebuilt board", ply, g)
                rows = e.tree_dump(g, agent)
                run.add(Tree(rows, root, agent, ply, slot, (ply, g)))
                last = slot // sb == (len(games) - 1) // sb
                run.slots.update(["slot first in block"] * (slot % sb == 0) +
                                 ["slot last in block"] * (slot % sb == sb - 1) + ["slot in last block"] * last +
                                 ["last block partial"] * (last and len(games) % sb != 0))
        if n_active == 0:
            break
    e.arena_finish()
    e.close()
    return run, twin


def random_complete_game(c, rng, n_moves):
    g = new_game(c)
    for i in range(n_moves):
        p = R.BLACK if i % 2 == 0 else R.WHITE
        legal = [mv for mv in range(c.m * c.n) if g.board[mv] == 0 and g.check(p, mv)]
        g = g.apply(p, int(rng.choice(legal)))
    return g


def collect_external(lib, c):
    e, twin = make_engines(lib, c)
    run = Run(c, lib)
    rng = np.random.default_rng(c.seed)
    for agent in (0, 1):
        g = random_complete_game(c, rng, c.plies + agent)
        player = R.BLACK if len(g.history) % 2 == 0 else R.WHITE
        assert len(g.historical) >= 8
        e.search(agent, g.board, player, player, move_number=len(g.history), passes=g.n_passes,
                 hist=np.array(g.historical, np.int32), last_move=g.history[-1][1], ko=g.ko)
        root = g.clone()
        root.next = player
        run.add(Tree(e.tree_dump(0, agent), root, agent, 0, 0, ("external", agent)))
    e.close()
    return run, twin


# ---------------------------------------------------------------------------------------------------------------------
def restate_priors(pol, moves, L, fault=None):
    """k_expand_backup's prior list: moves in index order then Pass, Pass's entry pol[L-1], legalSum in list order,
    normalised, stable descending sort.  Returns (moves, priors) in the node's child order."""
    lst = sorted(moves, key=lambda mv: (mv == R.PASS, mv))
    pass_entry = L - 2 if fault == "pass-entry" else L - 1
    vals = np.array([pol[pass_entry] if mv == R.PASS else pol[mv] for mv in lst], np.float32)
    s = f32(0)
    for v in (np.sort(vals)[::-1] if fault == "sorted-legalsum" else vals):
        s = f32(s + v)
    if s > TINY:
        p = vals / s
    else:
        p = np.full(len(vals), f32(1) / f32(len(vals)), np.float32)
    order = np.argsort(-p, kind="stable")
    return [lst[i] for i in order], p[order]


def seq_sum(v, k):
    w = f32(0)
    for _ in range(k):
        w = f32(w + v)
    return w


def audit(run, outs, fault=None):
    """Checks every audited tree against the twin's outputs; returns (mismatching nodes, counts)."""
    c = run.c
    L = action_space(c) + 1
    term_max = 2.0 + ((c.m * c.n + abs(c.komi)) if c.kind == K.GAME_WQ else 0.0)  # |v'| < 2; a two-pass score
    bad, n = [], collections.Counter()
    partner = run.partners() if fault == "neighbour-slot" else {}
    for t in run.trees:
        rows = t.rows
        N = rows[:, 2].astype(np.int64)
        W = rows[:, 3].copy().view(np.float32)
        src = dict(t.idx)
        if fault == "parent-position":
            src = {i: t.idx[t.parent[i]] if i else t.idx[i] for i in t.expanded}
        if fault == "sibling-swap":
            for p in t.expanded:
                ex = [k for k in t.kids.get(p, []) if rows[k, 5]]
                for a, b in zip(ex[0::2], ex[1::2]):
                    src[a], src[b] = src[b], src[a]
        if partner.get(id(t)) is not None:  # each expanded node reads the neighbouring game's node of the same rank
            q = partner[id(t)]
            for i, j in zip(t.expanded, q.expanded):
                src[i] = q.idx[j]
        n["unexpanded N > 1 (terminal scores)"] += int(((rows[:, 5] == 0) & (N > 1)).sum())
        for i in t.expanded:
            pol, v = outs[t.agent][0][src[i]], outs[t.agent][1][src[i]]
            kids = t.kids.get(i, [])
            want_moves, want_p = restate_priors(pol, [int(rows[k, 1]) for k in kids], L, fault)
            got_moves, got_p = [int(rows[k, 1]) for k in kids], rows[kids, 4].astype(np.uint32)
            if i == 0:  # bestMove re-sorted the root's children: compare the prior of every move
                ok = dict(zip(got_moves, got_p)) == dict(zip(want_moves, want_p.view(np.uint32)))
            else:
                ok = got_moves == want_moves and (got_p == want_p.view(np.uint32)).all()
            to_move = t.states[i].next
            vp = v if (to_move == R.BLACK or fault == "no-white-flip") else f32(f32(1) - v)
            k = int(N[i] - 1 - sum(N[j] - 1 for j in kids))
            n["expanded"] += 1
            n["to move %s" % ("black" if to_move == R.BLACK else "white")] += 1
            n["agent %d" % t.agent] += 1
            n["depth >= 2"] += int(rows[i, 0] >= 2)
            if i:
                n["k >= 2"] += int(k >= 2)
                if all(N[j] == 1 for j in kids):
                    n["leaf values"] += 1
                    ok &= k >= 1 and f32(W[i]).view(np.uint32) == seq_sum(vp, k).view(np.uint32)
                else:
                    n["internal values"] += 1
                    dev = abs(float(W[i]) - math.fsum([float(W[j]) for j in kids] + [k * float(vp)]))
                    bound = U * term_max * (N[i] * (N[i] - 1) + sum(N[j] * (N[j] - 1) for j in kids))
                    ok &= k >= 0 and dev <= bound
            if not ok:
                bad.append((t.label, i))
    return bad, n


def check_legal_children(run, per_tree=2):
    """The children of a few expanded nodes per tree are exactly the legal moves of the rebuilt position."""
    checked = 0
    for t in run.trees:
        for i in t.expanded[1:per_tree + 1]:
            s = t.states[i]
            want = {mv for mv in range(s.action_space()) if s.check(s.next, mv)}
            if run.c.kind != K.GAME_MNK:
                want.add(R.PASS)
            assert {int(t.rows[k, 1]) for k in t.kids.get(i, [])} == want, (run.c.name, t.label, i)
            checked += 1
    return checked


def same_bits(x, y):
    return all((a.view(np.uint32) == b.view(np.uint32)).all() for a, b in zip(x, y))


def check_batch_position(run, twin, outs):
    """az_infer gives each row the same bits wherever it sits in the batch: reversed, shifted by one slot, alone."""
    sb = heads_block(slot_count(run.c))
    for a in (0, 1):
        if outs[a] is None:
            continue
        P = np.array(run.planes[a], np.float32)
        p0, v0 = outs[a]
        pr, vr = twin.infer(a, P[::-1])
        assert same_bits((pr[::-1], vr[::-1]), (p0, v0)), (run.c.name, "reversed")
        assert same_bits(twin.infer(a, P[1:]), (p0[1:], v0[1:])), (run.c.name, "shifted")
        for r in sorted({0, sb - 1, sb, len(P) - 1}):
            if r < len(P):
                assert same_bits(twin.infer(a, P[r:r + 1]), (p0[r:r + 1], v0[r:r + 1])), (run.c.name, "alone", r)


def heads_vs_float64(run, twin, outs, rows=48):
    """The float64 heads on the twin's tower output, on up to `rows` distinct audited planes per agent spread over the
    whole audit; returns the worst policy (relative) and value (absolute) deviation and the rows compared."""
    worst_p = worst_v = 0.0
    compared = 0
    for a in (0, 1):
        if outs[a] is None:
            continue
        P = np.array(run.planes[a], np.float32)
        first = np.sort(np.unique(P, axis=0, return_index=True)[1])
        pick = first[np.linspace(0, len(first) - 1, min(rows, len(first))).astype(int)]
        tower = twin.infer_tower(a, P[pick]).astype(np.float64)
        p_ref, v_ref = D.Net(D.unpack(twin, a), run.c.layers).infer(tower=tower)
        worst_p = max(worst_p, float((np.abs(outs[a][0][pick] - p_ref) / p_ref).max()))
        worst_v = max(worst_v, float(np.abs(outs[a][1][pick] - v_ref).max()))
        compared += len(pick)
    return worst_p, worst_v, compared


def report(c, n, extra=""):
    print("%s: %s%s" % (c.name, ", ".join("%s %d" % kv for kv in sorted(n.items())), extra))


def assert_coverage(run, n, outs):
    c = run.c
    shared = bool(c.flags & K.FLAG_SHARED_TREE)
    assert n["expanded"] > 0 and n["leaf values"] > 0 and n["depth >= 2"] > 0, (c.name, n)
    assert n["to move black"] > 0 and n["to move white"] > 0, (c.name, n)
    assert n["agent 0"] > 0 and (shared or n["agent 1"] > 0), (c.name, n)
    if c.workers > 1:
        assert n["k >= 2"] > 0, (c.name, n)
    if c.audit is not None:
        assert run.slots["slot first in block"] > 0 and run.slots["slot last in block"] > 0, (c.name, run.slots)
        assert run.slots["slot in last block"] > 0, (c.name, run.slots)
    if c.games > 1:  # games in neighbouring slots hold different positions, so a slot mix-up changes what is read
        diff, pairs = run.distinct_neighbours()
        assert pairs > 0 and diff >= 0.75 * pairs, (c.name, diff, pairs)
        assert audit(run, outs, "neighbour-slot")[0], c.name
    if c.pass_logit:  # games ended by two passes at different plies: the audited waves ran on shrinking batches
        assert any(0 < a < c.games for a in run.active[c.first:]), (c.name, run.active)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the auditor is right (the oracle audits clean) and sharp (each restated fault fails it)
@pytest.fixture(scope="module")
def oracle_runs(oracle):
    runs = []
    for c in CPU_CASES:
        run, twin = collect_arena(oracle, c)
        runs.append((run, twin, run.evaluate(twin)))
    yield runs
    for _, twin, _ in runs:
        twin.close()


@pytest.mark.parametrize("ci", range(len(CPU_CASES)), ids=[c.name for c in CPU_CASES])
def test_oracle_audits_clean(oracle_runs, ci):
    run, twin, outs = oracle_runs[ci]
    bad, n = audit(run, outs)
    legal = check_legal_children(run)
    check_batch_position(run, twin, outs)
    report(run.c, n, ", children legality checked at %d nodes" % legal)
    assert not bad, (run.c.name, len(bad), bad[:5])
    assert_coverage(run, n, outs)
    if run.c.kind == K.GAME_WQ:  # every history plane filled at the last plies' roots
        assert max(len(t.states[0].history) for t in run.trees) >= 9
    if run.c.kind == K.GAME_MNK:  # tree reuse: nodes created by an earlier search sit below later roots
        assert max(int(t.rows[0, 2]) for t in run.trees) > run.c.sims + 1


def test_each_fault_fails_the_audit(oracle_runs):
    """The auditor catches each slip the wave could make, in every case where the slip changes what is read or stored
    (fault_applies): history planes one ply stale, every node encoded at its parent's position, no White flip of the
    value, two siblings' outputs exchanged, the outputs of the games in neighbouring slots exchanged (a slot mix-up),
    the Pass prior read from the wrong entry, legalSum summed in sorted order."""
    missed = []
    for fault in FAULTS:
        per_case = []
        for run, twin, outs in oracle_runs:
            o = run.evaluate(twin, stale=True) if fault == "stale-history" else outs
            per_case.append(len(audit(run, o, fault)[0]))
            if fault_applies(fault, run.c) and not per_case[-1]:
                missed.append((fault, run.c.name))
        print("fault %-16s mismatching nodes per case %s" % (fault, per_case))
    assert not missed, missed


def test_gpu_cases_cover_the_production_configurations():
    """The GPU cases reach every heads block size, every tower kernel family, workers, the shared tree, the complete
    rules, tree reuse and the external search, by the dispatch rules restated above."""
    seen = set()
    for c in GPU_CASES + [EXTERNAL]:
        gs = slot_count(c)
        seen.add(heads_kernel(c, gs))
        seen.add(tower_family(c))
        if c.workers > 1:
            seen.add("workers")
        if c.flags & K.FLAG_SHARED_TREE:
            seen.add("shared tree")
        if c.flags & K.FLAG_WQ_COMPLETE:
            seen.add("complete rules")
        if c.kind == K.GAME_MNK and c.plies >= 3:
            seen.add("tree reuse")
        if c.m != c.n:
            seen.add("H != W")
    seen.add("external")
    print(sorted(seen))
    c3, c3w = GPU_CASES[0], GPU_CASES[1]
    assert heads_block(slot_count(c3)) == 4 and slot_count(c3) == 1024
    assert heads_block(slot_count(c3w)) == 8 and slot_count(c3w) == 1088
    assert 8 * (3 * 361 + 362 + 512) * 4 > 48 * 1024  # SB = 8 at 19x19 / FC 512 needs the opt-in shared memory
    want = {"k_heads_tiled<1>", "k_heads_tiled<2>", "k_heads_tiled<4>", "k_heads_tiled<8>", "k_heads_f32",
            "k_conv3x3_m192 per-sample", "k_conv3x3_m192 flat", "k_conv3x3_tc flat", "k_net_small", "k_smallnet_fp16",
            "fp32 k_unit_f32", "workers", "shared tree", "complete rules", "tree reuse", "H != W", "external"}
    assert want <= seen, want - seen


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("c", GPU_CASES + [EXTERNAL], ids=[c.name for c in GPU_CASES + [EXTERNAL]])
def test_tree_audit_on_device(engine_lib, c):
    run, twin = (collect_external if c is EXTERNAL else collect_arena)(engine_lib, c)
    outs = run.evaluate(twin)
    bad, n = audit(run, outs)
    legal = check_legal_children(run)
    check_batch_position(run, twin, outs)
    wp, wv, rows = heads_vs_float64(run, twin, outs)
    twin.close()
    distinct = sum(len(np.unique(np.array(p, np.float32), axis=0)) for p in run.planes if p)
    report(c, n, ", %s, %s, children legality checked at %d nodes, slots %s, distinct planes %d, neighbour pairs "
           "differing %d of %d, games moving per ply %s ; heads vs float64 on %d rows: policy rel %.3g, value abs %.3g"
           % (tower_family(c), heads_kernel(c, slot_count(c)), legal, dict(run.slots), distinct,
              *run.distinct_neighbours(), run.active, rows, wp, wv))
    assert not bad, (c.name, len(bad), bad[:5])
    assert_coverage(run, n, outs)
    assert wp <= TOL_POLICY and wv <= TOL_VALUE, (c.name, wp, wv)
