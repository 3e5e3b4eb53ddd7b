"""Search without the host (elfb200_mcts_*_dev, MctsBatch.search_dev / choose_dev / results_dev / advance_dev /
reset_dev): the device forms compute exactly what the host forms compute.

CPU: the kernels run on the SIMT emulator build of the kernel sources (tests/simt_emu), under every lane order.
Two search handles run in lockstep on two identical boards.  One is driven by the host forms (begin_move with its
host move counter k, select / expand_backup, choose with seed s ^ k, results, advance, reset); the other by the
device forms through the product's MctsBatch methods, lent to the emulator's search class (they only use the handle
and the library, with CPU tensors for device memory), with the move index k and the seed
s ^ k in tensors.  Each board is driven through GoEnv: a game that ends on the board restarts by itself, a resigned
game is restarted and its tree reset.  Every move both handles give equal actions, values, results tables, root
edges, tree usage, error and statistics counters, and the boards stay equal.  The runs contain root noise, sampled
moves, resignations, games that end on the board, pruned trees and inactive games, and assert each of them.
tests/test_zz_gpu_search_dev.py runs the device forms on an H100, eagerly and replayed from a CUDA graph."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from elf_b200 import lib as _l
from elf_b200.env import GoEnv
from elf_b200.mcts import MctsBatch
from tests import oracles

pytestmark = pytest.mark.timeout(1800)

ERR_ARG, ERR_STATE = -1, -3  # ELFB200_ERR_ARG / ELFB200_ERR_STATE (include/elfb200.h)
R = 32  # rollouts per move, whole waves of 8
# root noise on; a node pool of R + 8 slots per game, so persistent trees are pruned to fit it
OPTS = dict(num_rollouts=R, num_rollouts_per_batch=8, virtual_loss=1, persistent_tree=1, c_puct=1.5, seed=11,
            root_epsilon=0.25, root_alpha=0.03, nodes_per_game=R + 8)
CUTOFF = 30  # sample the move while ply <= 30
THRES = 0.9  # resign below a value of -0.1 (from ply 50 on)
SEED = 0x5EED_0000_C0FFEE  # the host form's seed of move k is SEED ^ k


# ---- SIMT emulator ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    from tests import emu as E

    try:
        E.emu_lib()
    except Exception as e:  # no g++ / ucontext: the emulator is a convenience, not a requirement
        pytest.skip(f"SIMT emulator build unavailable: {e}")
    return E


@pytest.fixture(params=["ascending", "reverse", "random"])
def lane_order(request, emu):
    """order in which the emulator runs the lanes of a warp between two collectives"""
    L = emu.emu_lib()
    L.simt_emu_set_order(["ascending", "reverse", "random"].index(request.param))
    yield request.param
    L.simt_emu_set_order(0)


# ---- scenario ---------------------------------------------------------------------------------------------
def random_game(n, plies, rng):
    """`plies` uniform random legal non-pass moves from the empty board (the C restatement of the rules), passing
    only when no point is legal; the game must not end on the way"""
    o = oracles.Oracle(n)
    moves = []
    for _ in range(plies):
        c = np.flatnonzero(o.legal()[: n * n])
        a = int(rng.choice(c)) if len(c) else n * n
        assert o.forward(a)
        moves.append(a)
        assert not o.terminated()
    return moves


def opening_lists(n, G, rng):
    """game 0 twelve plies before the ply cap (2 N^2: it never resigns and ends on the board), games 1 and 2 past
    ply 50 (game 1 may resign, game 2 never does), the others within the sampling cutoff"""
    lengths = [2 * n * n - 12, 52, 56] + [int(rng.integers(0, 12)) for _ in range(G - 3)]
    return [random_game(n, k, rng) for k in lengths]


_DEV_METHODS = ("search_dev", "choose_dev", "results_dev", "advance_dev", "reset_dev", "_check_dev", "_mask_dev",
                "_dev_call", "_dev_out")


def emu_search_class(emu):
    """the emulator's search class with the product's device-form methods"""
    return type("EmuDevSearch", (emu.EmuSearch,), {k: MctsBatch.__dict__[k] for k in _DEV_METHODS})


class Side:
    """one board (through GoEnv) and one search handle; `fmt` "f32" or "df" leaf planes"""

    def __init__(self, emu, n, lists, fmt, opts):
        self.gb = emu.emu_batch(len(lists), n)
        self.gb.replay(lists)
        self.env = GoEnv(self.gb, device="cpu")
        self.mc = emu_search_class(emu)(self.gb, **opts)
        if fmt == "df":
            mc = self.mc
            mc._fmt, mc.feat_key = _l.FEAT_DF_F32_NCHW, "s"
            mc.feat = torch.zeros((mc.max_leaves, 25, n, n), dtype=torch.float32)

    def close(self):
        self.mc.close()
        self.gb.close()


def make_net(kind, n):
    """(host reply, device reply) builders.  "hash": oracles.fakenet keyed by the leaf hash of the host handle's
    leaves, handed to the device rows that hold the same planes; "plane" / "df": the plane-digest nets on each
    handle's own planes, all max_leaves rows on the device side."""
    P1 = n * n + 1
    if kind == "hash":
        def host(mc, s):
            pi, v = oracles.fakenet(mc.leaf_info()[0], P1)
            return torch.from_numpy(pi), torch.from_numpy(v)
        return host, None
    if kind == "plane":
        from tests.planenet import PlaneNet

        net = PlaneNet(n, "cpu", batchsize=0)
    else:
        from tests.df_search import DfNet

        net = DfNet(n, "cpu")

    def reply(mc, s):
        r = net({"s": s})
        return r["pi"], r["V"]
    return reply, reply


def bits(t):
    return t.contiguous().numpy().view(np.uint8)


def assert_same_move(H, D, k, tables_d, label):
    """everything a move leaves behind is equal on both handles"""
    rh = H.results()
    for key, t in tables_d.items():
        assert rh[key].tobytes() == t.numpy().tobytes(), f"results {key}, move {k} {label}"
    eh, ed = H.root_edges(), D.root_edges()
    for key in eh:
        assert eh[key].tobytes() == ed[key].tobytes(), f"root edges {key}, move {k} {label}"
    for a, b in zip(MctsBatch.tree_usage(H), MctsBatch.tree_usage(D)):
        assert (a == b).all(), f"tree usage, move {k} {label}"
    assert (H.errors() == D.errors()).all(), (H.errors(), D.errors(), k, label)
    assert (H.stats() == D.stats()).all(), (H.stats(), D.stats(), k, label)


def run_lockstep(emu, n, G, moves, kind="hash", fmt="f32", opts=OPTS, seed=1):
    """`moves` moves of both handles in lockstep; returns the event counts"""
    rng = np.random.default_rng(seed + n)
    lists = opening_lists(n, G, rng)
    hs, ds = Side(emu, n, lists, fmt, opts), Side(emu, n, lists, fmt, opts)
    H, D = hs.mc, ds.mc
    host_net, dev_net = make_net(kind, n)
    ev = dict(noise=0, sampled=0, resigned=0, ended=0, inactive=0)
    nr = np.zeros(G, np.uint8)
    nr[[0, 2]] = 1
    move = torch.zeros(1, dtype=torch.int64)
    for k in range(moves):
        active = np.ones(G, np.uint8)
        if k % 4 == 3:
            active[G - 1] = 0
        p0 = H.root_priors()
        H.begin_move(active)
        p1 = H.root_priors()
        ev["noise"] += int(((p0 >= 0) & (p0 != p1)).any(1).sum())

        def actor(batch):
            s = H.select()
            m = s.shape[0]
            x = batch[D.feat_key]
            assert x.shape[0] == D.max_leaves
            # leaves take their rows in the order the games claim them (an atomic counter), which differs between
            # the handles under the random lane order: the device rows are the host rows, permuted
            hrows = [bits(s[i]).tobytes() for i in range(m)]
            drows = [bits(x[i]).tobytes() for i in range(m)]
            assert sorted(drows) == sorted(hrows), f"leaf planes of a wave, move {k}"
            at = {b: i for i, b in enumerate(hrows)}
            perm = torch.tensor([at[b] for b in drows], dtype=torch.int64)
            if m == 0:
                H.expand_backup(None, None)
            else:
                pi, v = host_net(H, s)
                H.expand_backup(pi, v)
            if dev_net is not None:
                return dict(zip(("pi", "V"), dev_net(D, x)))
            P = torch.zeros((D.max_leaves, n * n + 1), dtype=torch.float32)
            V = torch.zeros(D.max_leaves, dtype=torch.float32)
            if m:
                P[:m], V[:m] = pi[perm], v[perm]
            return {"pi": P, "V": V}

        D.search_dev(actor, move, torch.from_numpy(active).bool())
        ply = hs.gb.info()[:, 0]
        ah, vh = H.choose(CUTOFF, THRES, nr, seed=SEED ^ k)
        ad, vd = D.choose_dev(CUTOFF, THRES, torch.tensor([SEED ^ k]), torch.from_numpy(nr))
        assert (ah == ad.numpy()).all(), (k, ah, ad)
        assert vh.tobytes() == vd.numpy().tobytes(), (k, vh, vd)
        assert_same_move(H, D, k, D.results_dev(), f"n={n} {kind}")
        ev["sampled"] += int(((ply <= CUTOFF) & (ah >= 0)).sum())
        ev["resigned"] += int((ah == -1).sum())
        ev["inactive"] += int((ah == -2).sum())
        # host: play, restart resigned games, advance, reset the trees of the games that ended
        obs = hs.env.step(torch.from_numpy(ah))
        done = obs["done"].numpy().astype(bool)
        resigned = ah == -1
        hs.env.reset(torch.from_numpy(resigned))
        H.advance(ah)
        H.reset((done | resigned).astype(np.uint8))
        ev["ended"] += int(done.sum())
        # device: the README's loop
        obs = ds.env.step(ad)
        res_t = ad == -1
        ended = obs["done"].bool() | res_t  # read before reset(), which clears done
        ds.env.reset(res_t)
        D.advance_dev(ad)
        D.reset_dev(ended)
        move.add_(1)
        assert (hs.gb.info() == ds.gb.info()).all(), f"board info after move {k}"
        assert (hs.gb.getHashCode() == ds.gb.getHashCode()).all(), f"hashes after move {k}"
    e = H.errors()
    assert e[0] == 0 and e[1] == 0 and e[2] == 0, e
    ev["pruned"] = int(e[3])
    for x in (hs, ds):
        x.close()
    return ev


def assert_every_event(ev):
    for k in ("noise", "sampled", "resigned", "ended", "inactive", "pruned"):
        assert ev[k] > 0, (k, ev)


@pytest.mark.parametrize("n,G", [(9, 4), (19, 4)])
def test_device_forms_equal_host_forms(emu, lane_order, n, G):
    """fakenet keyed by the leaf hash, rotation_flip on, f32 planes: 40 moves"""
    assert_every_event(run_lockstep(emu, n, G, 40))


@pytest.mark.parametrize("kind,fmt", [("plane", "f32"), ("df", "df")])
def test_device_forms_equal_host_forms_on_planes(emu, kind, fmt):
    """the nets keyed by the planes each handle hands them (the device side evaluates all max_leaves rows): the
    AGZ planes with the plane-digest net and the DarkForest planes with the DF digest, 9x9"""
    assert_every_event(run_lockstep(emu, 9, 4, 40, kind=kind, fmt=fmt))


# ---- refused calls ---------------------------------------------------------------------------------------
def test_refused_calls(emu):
    """each refusal returns its code, enqueues nothing, and the handle searches on as its twin afterwards"""
    L = emu.emu_lib()
    n, G = 9, 3
    lists = [random_game(n, k, np.random.default_rng(k)) for k in (3, 8, 0)]
    hs, ds = Side(emu, n, lists, "f32", OPTS), Side(emu, n, lists, "f32", OPTS)
    H, D, m = hs.mc, ds.mc, ds.mc._m
    buf = lambda dt, k: np.zeros(k, dt)  # noqa: E731
    feat, pi, v = D.feat.data_ptr(), buf(np.float32, D.max_leaves * (n * n + 1)), buf(np.float32, D.max_leaves)
    mv, act = buf(np.int64, 1), buf(np.int32, G)

    def refused(rc_expected, fn, *args):
        n0 = ds.gb.launch_count()
        assert fn(*args) == rc_expected, (fn, L.elfb200_last_error())
        assert ds.gb.launch_count() == n0

    refused(ERR_ARG, L.elfb200_mcts_reset_dev, None, None)
    refused(ERR_ARG, L.elfb200_mcts_begin_move_dev, None, None, mv.ctypes.data)
    refused(ERR_ARG, L.elfb200_mcts_begin_move_dev, m, None, None)  # root noise is on
    refused(ERR_ARG, L.elfb200_mcts_select_dev, None, feat, _l.FEAT_F32_NCHW, 0)
    refused(ERR_ARG, L.elfb200_mcts_select_dev, m, None, _l.FEAT_F32_NCHW, 0)
    refused(ERR_ARG, L.elfb200_mcts_select_dev, m, feat, 7, 0)
    refused(ERR_ARG, L.elfb200_mcts_select_dev, m, feat, _l.FEAT_F16_NHWC, 20)
    refused(ERR_STATE, L.elfb200_mcts_expand_backup_dev, m, pi.ctypes.data, v.ctypes.data)  # no wave open
    refused(ERR_ARG, L.elfb200_mcts_results_dev, None, None, None, None, None, None)
    refused(ERR_ARG, L.elfb200_mcts_choose_dev, m, 0, 0.0, None, None, act.ctypes.data, None)
    refused(ERR_ARG, L.elfb200_mcts_choose_dev, m, 0, 0.0, None, mv.ctypes.data, None, None)
    refused(ERR_ARG, L.elfb200_mcts_advance_dev, m, None)
    # an open wave: no second select, no new move
    _l.check(L, L.elfb200_mcts_begin_move_dev(m, None, mv.ctypes.data))
    _l.check(L, L.elfb200_mcts_select_dev(m, feat, _l.FEAT_F32_NCHW, 0))
    refused(ERR_STATE, L.elfb200_mcts_select_dev, m, feat, _l.FEAT_F32_NCHW, 0)
    refused(ERR_STATE, L.elfb200_mcts_begin_move_dev, m, None, mv.ctypes.data)
    refused(ERR_ARG, L.elfb200_mcts_expand_backup_dev, m, None, v.ctypes.data)
    # finish the move on both handles: the host handle's counter is at 1 after this move, the device's tensor too
    H.begin_move()
    for w in range(D.waves_per_move):
        s = H.select()
        if s.shape[0]:
            p, val = oracles.fakenet(H.leaf_info()[0], n * n + 1)
            H.expand_backup(torch.from_numpy(p), torch.from_numpy(val))
            pi[: p.size] = p.reshape(-1)
            v[: val.size] = val
        else:
            H.expand_backup(None, None)
        if w:
            _l.check(L, L.elfb200_mcts_select_dev(m, feat, _l.FEAT_F32_NCHW, 0))
        _l.check(L, L.elfb200_mcts_expand_backup_dev(m, pi.ctypes.data, v.ctypes.data))
    assert_same_move(H, D, 0, D.results_dev(), "after the refused calls")
    # a reference D4 stream: every device form is refused until it is cleared
    D.set_d4_stream(np.zeros((G, R), np.uint8))
    refused(ERR_STATE, L.elfb200_mcts_reset_dev, m, None)
    refused(ERR_STATE, L.elfb200_mcts_begin_move_dev, m, None, mv.ctypes.data)
    refused(ERR_STATE, L.elfb200_mcts_select_dev, m, feat, _l.FEAT_F32_NCHW, 0)
    refused(ERR_STATE, L.elfb200_mcts_expand_backup_dev, m, pi.ctypes.data, v.ctypes.data)
    refused(ERR_STATE, L.elfb200_mcts_results_dev, m, None, None, None, None, None)
    refused(ERR_STATE, L.elfb200_mcts_choose_dev, m, 0, 0.0, None, mv.ctypes.data, act.ctypes.data, None)
    refused(ERR_STATE, L.elfb200_mcts_advance_dev, m, act.ctypes.data)
    assert b"D4 stream" in L.elfb200_last_error()
    D.set_d4_stream(None)
    # the Python layer validates its tensors
    with pytest.raises(ValueError):
        D.search_dev(None, torch.zeros(1, dtype=torch.int32))
    with pytest.raises(ValueError):
        D.choose_dev(0, 0.0, torch.zeros(2, dtype=torch.int64))
    with pytest.raises(ValueError):
        D.advance_dev(torch.zeros(G, dtype=torch.int64))
    with pytest.raises(ValueError):
        D.reset_dev(torch.zeros(G + 1, dtype=torch.uint8))
    # and the handle carries on as its twin
    mv[0] = 1
    a = np.array([int(x) for x in H.results()["best_action"]], np.int32)
    for side in (hs, ds):
        side.gb.forward(a)
    H.advance(a)
    D.advance_dev(torch.from_numpy(a))

    def actor(batch):
        s = H.select()
        if s.shape[0] == 0:
            H.expand_backup(None, None)
            return {"pi": torch.zeros((D.max_leaves, n * n + 1)), "V": torch.zeros(D.max_leaves)}
        p, val = oracles.fakenet(H.leaf_info()[0], n * n + 1)
        H.expand_backup(torch.from_numpy(p), torch.from_numpy(val))
        P, V = torch.zeros((D.max_leaves, n * n + 1)), torch.zeros(D.max_leaves)
        P[: len(p)], V[: len(p)] = torch.from_numpy(p), torch.from_numpy(val)
        return {"pi": P, "V": V}

    H.begin_move()
    D.search_dev(actor, torch.from_numpy(mv))
    assert_same_move(H, D, 1, D.results_dev(), "the move after")
    for x in (hs, ds):
        x.close()


# ---- AddressSanitizer -------------------------------------------------------------------------------------
_ASAN_CHILD = r"""
import sys
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests/simt_emu")
import build
from elf_b200 import lib as _l
from tests import emu as E
E._lib = _l.load_library(build.build(asan=True))
from tests.test_search_dev import assert_every_event, run_lockstep
run_lockstep(E, 9, 4, 12)
run_lockstep(E, 19, 4, 6)
run_lockstep(E, 9, 4, 6, kind="df", fmt="df")
print("ASAN SEARCH DEV CLEAN")
"""


def test_lockstep_clean_under_address_sanitizer(emu):
    """the lockstep loop on the emulator build under AddressSanitizer (every device buffer is a heap allocation
    there, so any read or write outside a buffer is reported)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        asan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        pytest.skip(f"no gcc: {e}")
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("libasan is not installed")
    env = dict(os.environ, LD_PRELOAD=os.path.realpath(asan), ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0")
    r = subprocess.run([sys.executable, "-c", _ASAN_CHILD, root], env=env, capture_output=True, text=True, timeout=1700)
    assert r.returncode == 0 and "ASAN SEARCH DEV CLEAN" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]
