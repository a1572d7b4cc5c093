"""ctypes binding of include/agogo_b200.h.

The same header is exported by the product library (agogo_b200/libagogo_b200.so, CUDA) and by
the test-only CPU oracle; `load(path)` binds whichever shared object it is given.  This module
never chooses the oracle by itself: `load()` without a path is the product library and raises
if it has not been built.
"""
import ctypes as C
import os

import numpy as np

AZ_OK = 0
NONE, BLACK, WHITE = 0, 1, 2
PASS, RESIGN = -1, -2
GAME_MNK, GAME_C4, GAME_WQ = 0, 1, 2
ENC_TWO_PLANE, ENC_WQ18 = 0, 1
INF_DUAL, INF_DUMMY, INF_TABLE = 0, 1, 2
FLAG_SHARED_TREE, FLAG_FP32_TOWER, FLAG_FAST_TOWER, FLAG_WQ_COMPLETE = 1, 2, 4, 8
DONT_PREFER_PASS, PREFER_PASS, DONT_RESIGN = 0, 1, 2


class GameDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("m", C.c_int32), ("n", C.c_int32), ("k", C.c_int32),
                ("komi", C.c_float), ("max_moves", C.c_int32), ("zobrist_seed", C.c_uint64)]


class MCTSConfig(C.Structure):
    """mcts.Config (mcts/tree.go:15-29) + sims."""
    _fields_ = [("puct", C.c_float), ("timeout_ns", C.c_int64), ("m", C.c_int32), ("n", C.c_int32),
                ("random_count", C.c_int32), ("budget", C.c_int32), ("random_min_visits", C.c_uint32),
                ("random_temperature", C.c_float), ("dumb_pass", C.c_int32), ("resign_percentage", C.c_float),
                ("pass_preference", C.c_int32), ("sims", C.c_int32), ("workers", C.c_int32)]


class DualConfig(C.Structure):
    """dual.Config (dualnet/config.go:4-16)."""
    _fields_ = [("k", C.c_int32), ("shared_layers", C.c_int32), ("fc", C.c_int32), ("l2", C.c_double),
                ("batch_size", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("features", C.c_int32),
                ("action_space", C.c_int32), ("fwd_only", C.c_int32)]


class EngineDesc(C.Structure):
    _fields_ = [("game", GameDesc), ("mcts", MCTSConfig), ("nn", DualConfig), ("encoder", C.c_int32),
                ("n_games", C.c_int32), ("device", C.c_int32), ("flags", C.c_uint32), ("seed", C.c_uint64),
                ("act_scale_log2", C.c_int32), ("max_nodes_per_tree", C.c_int32)]


class State(C.Structure):
    _fields_ = [("board", C.POINTER(C.c_int32)), ("to_move", C.c_int32), ("move_number", C.c_int32), ("passes", C.c_int32),
                ("last_move", C.c_int32), ("n_hist", C.c_int32), ("hist", C.POINTER(C.c_int32)),
                ("n_moves", C.c_int32), ("moves", C.POINTER(C.c_int32)), ("ko", C.c_int32)]


class Counters(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("searches", "sims", "null_results", "evals", "select_children",
                                          "select_levels", "created", "backup_nodes", "kernel_launches")] + \
               [("reserved", C.c_uint64 * 7)]


SYMBOLS = [
    "az_engine_create", "az_engine_destroy", "az_last_error", "az_net_param_count", "az_net_param_desc",
    "az_net_init", "az_net_get_params", "az_net_set_params", "az_net_copy", "az_agent_set_inferer",
    "az_agent_set_table", "az_infer", "az_agent_stats", "az_agent_reset_stats", "az_arena_play", "az_arena_begin",
    "az_arena_step", "az_arena_finish", "az_search_begin", "az_search_run", "az_search_end", "az_game_record",
    "az_game_state", "az_examples_count", "az_examples_read", "az_examples_clear", "az_tree_dump", "az_rules_apply",
    "az_rules_status", "az_train", "az_comm_unique_id", "az_comm_init", "az_counters_get", "az_counters_reset",
    "az_build_info", "az_profile", "az_train_grads", "az_train_apply", "az_search", "az_comm_bench", "az_agent_reset_tree",
    "az_infer_tower",
]

_HERE = os.path.dirname(os.path.abspath(__file__))
PRODUCT_LIB = os.path.join(_HERE, "libagogo_b200.so")


class AZError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("az error %d: %s" % (code, msg))
        self.code = code


def _p(a, ct):
    return a.ctypes.data_as(C.POINTER(ct))


class Lib:
    def __init__(self, path):
        self.path = path
        self.dll = C.CDLL(path, mode=getattr(os, "RTLD_LOCAL", 0) | getattr(os, "RTLD_NOW", 2))
        d = self.dll
        d.az_last_error.restype = C.c_char_p
        d.az_last_error.argtypes = [C.c_void_p]
        d.az_build_info.restype = C.c_char_p
        d.az_engine_destroy.restype = None
        d.az_engine_destroy.argtypes = [C.c_void_p]
        for s in SYMBOLS:
            f = getattr(d, s)  # raises AttributeError if the library does not export it
            if s not in ("az_last_error", "az_build_info", "az_engine_destroy"):
                f.restype = C.c_int

    def build_info(self):
        return self.dll.az_build_info().decode()

    def create(self, desc):
        h = C.c_void_p()
        rc = self.dll.az_engine_create(C.byref(desc), C.byref(h))
        if rc != AZ_OK:
            raise AZError(rc, (self.dll.az_last_error(None) or b"").decode())
        return Engine(self, h, desc)


def load(path=None):
    """Bind a library exporting include/agogo_b200.h.  Default: the product CUDA library."""
    if path is None:
        path = PRODUCT_LIB
        if not os.path.exists(path):
            raise ImportError("agogo_b200: %s is not built — run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(there is no CPU fallback)" % path)
    return Lib(path)


class Engine:
    """Thin handle wrapper; one method per C entry point, numpy in/out."""

    def __init__(self, lib, handle, desc):
        self.lib, self.h, self.desc = lib, handle, desc
        g = desc.game
        self.cells = g.m * g.n
        self.action_space = g.n if g.kind == GAME_C4 else g.m * g.n  # State.ActionSpace()
        self.features = desc.nn.features
        self.plane = desc.nn.features * desc.nn.height * desc.nn.width
        self.A1 = desc.nn.action_space

    def close(self):
        if self.h:
            self.lib.dll.az_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != AZ_OK:
            raise AZError(rc, (self.lib.dll.az_last_error(self.h) or b"").decode())

    # ---- nets
    def param_count(self):
        nt, nf = C.c_int32(), C.c_uint64()
        self._ck(self.lib.dll.az_net_param_count(self.h, C.byref(nt), C.byref(nf)))
        return nt.value, nf.value

    def param_desc(self, i):
        name = C.create_string_buffer(96)
        shape = (C.c_int32 * 4)()
        rank, off, size = C.c_int32(), C.c_uint64(), C.c_uint64()
        self._ck(self.lib.dll.az_net_param_desc(self.h, i, name, shape, C.byref(rank), C.byref(off), C.byref(size)))
        return name.value.decode(), tuple(shape[:rank.value]), off.value, size.value

    def net_init(self, net, seed):
        self._ck(self.lib.dll.az_net_init(self.h, net, C.c_uint64(seed)))

    def net_get(self, net):
        n = self.param_count()[1]
        out = np.empty(n, np.float32)
        self._ck(self.lib.dll.az_net_get_params(self.h, net, _p(out, C.c_float), C.c_uint64(n)))
        return out

    def net_set(self, net, arr):
        arr = np.ascontiguousarray(arr, np.float32)
        self._ck(self.lib.dll.az_net_set_params(self.h, net, _p(arr, C.c_float), C.c_uint64(arr.size)))

    def net_copy(self, dst, src):
        self._ck(self.lib.dll.az_net_copy(self.h, dst, src))

    # ---- agents
    def set_inferer(self, agent, kind, dummy_player=0):
        self._ck(self.lib.dll.az_agent_set_inferer(self.h, agent, kind, dummy_player))

    def set_table(self, agent, rows, values):
        rows = np.ascontiguousarray(rows, np.float32)
        values = np.ascontiguousarray(values, np.float32)
        self._ck(self.lib.dll.az_agent_set_table(self.h, agent, rows.shape[0], rows.shape[1], _p(rows, C.c_float),
                                                 _p(values, C.c_float)))

    def infer(self, agent, planes):
        planes = np.ascontiguousarray(planes, np.float32).reshape(-1, self.plane)
        n = planes.shape[0]
        pol = np.empty((n, self.A1), np.float32)
        val = np.empty(n, np.float32)
        self._ck(self.lib.dll.az_infer(self.h, agent, _p(planes, C.c_float), n, _p(pol, C.c_float), _p(val, C.c_float)))
        return pol, val

    def infer_tower(self, agent, planes):
        """The residual tower's output for the same forward as infer(): [n, K, H, W] fp32 (diagnostics)."""
        planes = np.ascontiguousarray(planes, np.float32).reshape(-1, self.plane)
        n = planes.shape[0]
        nn = self.desc.nn
        out = np.empty((n, nn.k, nn.height, nn.width), np.float32)
        self._ck(self.lib.dll.az_infer_tower(self.h, agent, _p(planes, C.c_float), n, _p(out, C.c_float)))
        return out

    def stats(self, agent):
        w, l, d = C.c_float(), C.c_float(), C.c_float()
        self._ck(self.lib.dll.az_agent_stats(self.h, agent, C.byref(w), C.byref(l), C.byref(d)))
        return w.value, l.value, d.value

    def reset_stats(self, agent):
        self._ck(self.lib.dll.az_agent_reset_stats(self.h, agent))

    # ---- arena
    def arena_play(self, n_games, record):
        self._ck(self.lib.dll.az_arena_play(self.h, n_games, int(record)))

    def arena_begin(self, n_games, record):
        self._ck(self.lib.dll.az_arena_begin(self.h, n_games, int(record)))

    def arena_step(self):
        n = C.c_int32()
        self._ck(self.lib.dll.az_arena_step(self.h, C.byref(n)))
        return n.value

    def arena_finish(self):
        self._ck(self.lib.dll.az_arena_finish(self.h))

    def search_begin(self):
        self._ck(self.lib.dll.az_search_begin(self.h))

    def search_run(self, n):
        self._ck(self.lib.dll.az_search_run(self.h, n))

    def search_end(self):
        self._ck(self.lib.dll.az_search_end(self.h))

    def search(self, agent, board, to_move, player, move_number=0, passes=0, hist=None, last_move=-1, moves=None, ko=-1):
        """Agent.Search on an external position: returns (best move, visit counts by move, Pass last).  `moves` = the
        tail of the state's history as (player, move) pairs, oldest first (enables tree reuse across calls)."""
        board = np.ascontiguousarray(board, np.int32)
        hist = np.zeros((0, self.cells), np.int32) if hist is None else np.ascontiguousarray(hist, np.int32).reshape(-1, self.cells)
        mv = np.zeros((0, 2), np.int32) if moves is None else np.ascontiguousarray(moves, np.int32).reshape(-1, 2)
        st = State(_p(board, C.c_int32), to_move, move_number, passes, last_move, hist.shape[0], _p(hist, C.c_int32),
                   mv.shape[0], _p(mv, C.c_int32), ko)
        best = C.c_int32()
        visits = np.zeros(self.action_space + 1, np.float32)
        self._ck(self.lib.dll.az_search(self.h, agent, C.byref(st), player, C.byref(best), _p(visits, C.c_float)))
        return best.value, visits

    def reset_tree(self, agent):
        self._ck(self.lib.dll.az_agent_reset_tree(self.h, agent))

    def game_record(self, game, cap=4096):
        moves = np.empty(cap, np.int32)
        n, w, a, ne = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
        self._ck(self.lib.dll.az_game_record(self.h, game, _p(moves, C.c_int32), cap, C.byref(n), C.byref(w),
                                             C.byref(a), C.byref(ne)))
        return dict(moves=moves[:min(n.value, cap)].copy(), winner=w.value, a_player=a.value, n_examples=ne.value)

    def game_state(self, game):
        board = np.empty(self.cells, np.int32)
        tm, mn, ps, en, w = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
        self._ck(self.lib.dll.az_game_state(self.h, game, _p(board, C.c_int32), self.cells, C.byref(tm), C.byref(mn),
                                            C.byref(ps), C.byref(en), C.byref(w)))
        return dict(board=board, to_move=tm.value, move_number=mn.value, passes=ps.value, ended=en.value,
                    winner=w.value)

    def examples(self, clear=False):
        n = C.c_int64()
        self._ck(self.lib.dll.az_examples_count(self.h, C.byref(n)))
        n = n.value
        boards = np.empty((n, self.plane), np.float32)
        pols = np.empty((n, self.action_space + 1), np.float32)
        vals = np.empty(n, np.float32)
        if n:
            self._ck(self.lib.dll.az_examples_read(self.h, C.c_int64(0), C.c_int64(n), _p(boards, C.c_float),
                                                   _p(pols, C.c_float), _p(vals, C.c_float)))
        if clear:
            self._ck(self.lib.dll.az_examples_clear(self.h))
        return boards, pols, vals

    def tree_dump(self, game, tree, cap=1 << 16):
        while True:
            rows = np.empty((cap, 7), np.int32)
            n = C.c_int32()
            self._ck(self.lib.dll.az_tree_dump(self.h, game, tree, _p(rows, C.c_int32), cap, C.byref(n)))
            if n.value <= cap:
                return rows[:n.value].copy()
            cap = n.value

    # ---- rules
    def rules_apply(self, boards, players, moves):
        boards = np.ascontiguousarray(boards, np.int32).reshape(-1, self.cells)
        n = boards.shape[0]
        players = np.ascontiguousarray(players, np.int32)
        moves = np.ascontiguousarray(moves, np.int32)
        check = np.empty(n, np.int32)
        applied = np.empty(n, np.int32)
        taken = np.empty(n, np.int32)
        out = np.empty_like(boards)
        self._ck(self.lib.dll.az_rules_apply(self.h, n, _p(boards, C.c_int32), _p(players, C.c_int32),
                                             _p(moves, C.c_int32), _p(check, C.c_int32), _p(applied, C.c_int32),
                                             _p(out, C.c_int32), _p(taken, C.c_int32)))
        return check, applied, out, taken

    def rules_status(self, boards, passes=None):
        boards = np.ascontiguousarray(boards, np.int32).reshape(-1, self.cells)
        n = boards.shape[0]
        passes = np.zeros(n, np.int32) if passes is None else np.ascontiguousarray(passes, np.int32)
        ended = np.empty(n, np.int32)
        winner = np.empty(n, np.int32)
        sb = np.empty(n, np.float32)
        sw = np.empty(n, np.float32)
        self._ck(self.lib.dll.az_rules_status(self.h, n, _p(boards, C.c_int32), _p(passes, C.c_int32),
                                              _p(ended, C.c_int32), _p(winner, C.c_int32), _p(sb, C.c_float),
                                              _p(sw, C.c_float)))
        return ended, winner, sb, sw

    # ---- train
    def train(self, net, Xs, Pi, V, batches, iterations, lr=0.1, shuffle_seed=0):
        Xs = np.ascontiguousarray(Xs, np.float32)
        Pi = np.ascontiguousarray(Pi, np.float32)
        V = np.ascontiguousarray(V, np.float32)
        costs = np.empty(batches * iterations, np.float32)
        self._ck(self.lib.dll.az_train(self.h, net, _p(Xs, C.c_float), _p(Pi, C.c_float), _p(V, C.c_float), batches,
                                       iterations, C.c_float(lr), C.c_uint64(shuffle_seed), _p(costs, C.c_float)))
        return costs

    def train_grads(self, net, X, Pi, V):
        X = np.ascontiguousarray(X, np.float32)
        Pi = np.ascontiguousarray(Pi, np.float32)
        V = np.ascontiguousarray(V, np.float32)
        g = np.empty(self.param_count()[1], np.float32)
        c = C.c_float()
        self._ck(self.lib.dll.az_train_grads(self.h, net, _p(X, C.c_float), _p(Pi, C.c_float), _p(V, C.c_float),
                                             _p(g, C.c_float), C.byref(c)))
        return g, c.value

    def train_apply(self, net, grads, lr=0.1):
        grads = np.ascontiguousarray(grads, np.float32)
        self._ck(self.lib.dll.az_train_apply(self.h, net, _p(grads, C.c_float), C.c_float(lr)))

    def comm_init(self, rank, world, uid):
        buf = (C.c_uint8 * 128).from_buffer_copy(bytes(uid))
        self._ck(self.lib.dll.az_comm_init(self.h, rank, world, buf))

    def profile(self, enable):
        out = (C.c_double * 8)()
        self._ck(self.lib.dll.az_profile(self.h, int(enable), out))
        return dict(conv_ms=out[0], conv_launches=out[1], forward_ms=out[2], forward_calls=out[3], region_ms=out[4],
                    kernel_kind=int(out[5]))

    def comm_bench(self, net=1, iters=10):
        ms, nbytes = C.c_double(), C.c_double()
        self._ck(self.lib.dll.az_comm_bench(self.h, net, iters, C.byref(ms), C.byref(nbytes)))
        return ms.value, nbytes.value

    def counters(self):
        c = Counters()
        self._ck(self.lib.dll.az_counters_get(self.h, C.byref(c)))
        return {n: getattr(c, n) for n, _ in Counters._fields_ if n != "reserved"}

    def counters_reset(self):
        self._ck(self.lib.dll.az_counters_reset(self.h))


def comm_unique_id(lib):
    buf = (C.c_uint8 * 128)()
    rc = lib.dll.az_comm_unique_id(buf)
    if rc != AZ_OK:
        raise AZError(rc, "az_comm_unique_id")
    return bytes(buf)


def make_desc(kind, m, n, k=0, komi=0.0, sims=50, puct=1.0, nn=None, encoder=None, n_games=1, seed=1, flags=0,
              max_moves=0, device=0, zobrist_seed=12345, pass_preference=DONT_PREFER_PASS, dumb_pass=1,
              mcts_m=None, mcts_n=None, workers=0):
    """Build an EngineDesc the way the reference's programs build their Configs."""
    d = EngineDesc()
    d.game = GameDesc(kind, m, n, k, komi, max_moves, zobrist_seed)
    d.mcts = MCTSConfig(puct, 0, mcts_m if mcts_m is not None else m, mcts_n if mcts_n is not None else n, 0, 10000, 0,
                        0.0, dumb_pass, 0.0, pass_preference, sims, workers)
    cells = m * n
    A = n if kind == GAME_C4 else cells
    if nn is None:
        nn = dict(k=3, shared_layers=1, fc=4, batch_size=4)
    feats = nn.get("features", 18 if (encoder == ENC_WQ18 or (encoder is None and kind == GAME_WQ)) else 2)
    d.nn = DualConfig(nn["k"], nn["shared_layers"], nn["fc"], 0.0, nn.get("batch_size", 4), n, m, feats,
                      nn.get("action_space", A + 1), 0)
    d.encoder = encoder if encoder is not None else (ENC_WQ18 if kind == GAME_WQ else ENC_TWO_PLANE)
    d.n_games, d.device, d.flags, d.seed = n_games, device, flags, seed
    d.act_scale_log2, d.max_nodes_per_tree = 0, 0
    return d
