"""Search without the host on an H100: MctsBatch.search_dev / choose_dev / results_dev / advance_dev / reset_dev over
GoEnv, eagerly and replayed from a CUDA graph, against the host-driven loop on a GoBatch (tests/test_search_dev.py
runs the same lockstep on the SIMT emulator).  The network is tests/planenet.PlaneNet, keyed by the planes it is
handed, with rotation_flip on.
A: the device forms eagerly, move for move equal to the host forms (19x19 at G = 512, 9x9 at G = 2048).
B: one whole move (the README's az_move) captured in a CUDA graph and replayed, in the f32 and f16 leaf formats.
C: the random draws of a replayed graph follow the device counters."""
import time

import numpy as np
import pytest
import torch

from elf_b200 import GoBatch
from elf_b200.env import GoEnv
from elf_b200.mcts import MctsBatch
from tests.planenet import PlaneNet
from tests.test_search_dev import CUTOFF, OPTS, SEED, THRES, random_game

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = 0
OPTS = dict(OPTS, num_rollouts=64, nodes_per_game=64 + 8)  # 64 rollouts per move, a pool that prunes trees


@pytest.fixture(autouse=True)
def report():
    """wall time and device memory of each test, printed for the record"""
    torch.cuda.init()
    torch.cuda.reset_peak_memory_stats(DEV)
    t0 = time.perf_counter()
    yield
    free, total = torch.cuda.mem_get_info(DEV)
    print(f"\n[search_dev] {time.perf_counter() - t0:.1f} s, {(total - free) / 1e9:.1f} GB device memory in use at the "
          f"end, {torch.cuda.max_memory_allocated(DEV) / 1e9:.2f} GB max_memory_allocated")


def openings(n, G, seed):
    """8 games a few plies before the ply cap (they end on the board), 8 past ply 50 (they may resign), the others
    within the sampling cutoff"""
    rng = np.random.default_rng(seed)
    long = [random_game(n, 2 * n * n - 6 - (g % 4), rng) for g in range(8)]
    mid = [random_game(n, 52 + g, rng) for g in range(8)]
    return long + mid + [random_game(n, int(rng.integers(0, 12)), rng) for _ in range(G - 16)]


NEVER_RESIGN = 4  # the first four long games never resign: they reach the ply cap


class Host:
    """the host-driven loop: GoBatch, MctsBatch.begin_move / wave / choose / results / advance / reset"""

    def __init__(self, n, lists, net, fmt):
        self.gb = GoBatch(len(lists), board_size=n, device=DEV)
        self.gb.replay(lists)
        self.mc = MctsBatch(self.gb, feature_format=fmt, **OPTS)
        self.net, self.k = net, 0
        self.nr = np.zeros(len(lists), np.uint8)
        self.nr[:NEVER_RESIGN] = 1

    def move(self, active):
        mc = self.mc
        p0 = mc.root_priors()
        mc.begin_move(active)
        noised = int(((p0 >= 0) & (p0 != mc.root_priors())).any(1).sum())
        for _ in range(mc.waves_per_move):
            mc.wave(self.net)
        ply = self.gb.info()[:, 0]
        a, v = mc.choose(CUTOFF, THRES, self.nr, seed=SEED ^ self.k)
        r = mc.results()
        r.update(actions=a, values=v, noised=noised, sampled=int(((ply <= CUTOFF) & (a >= 0)).sum()))
        self.gb.forward(a)
        done = self.gb.terminated()
        ended = (done | (a == -1)).astype(np.uint8)
        self.gb.reset(ended)
        mc.advance(a)
        mc.reset(ended)
        r.update(ended=int(done.sum()), after=after_move(mc, self.gb))
        self.k += 1
        return r


def after_move(mc, gb):
    """what a move leaves behind: root edges, tree usage, counters, boards"""
    return dict(edges=mc.root_edges(), usage=mc.tree_usage(), errors=mc.errors(), stats=mc.stats(), info=gb.info(),
                hash=gb.getHashCode())


class Device:
    """GoEnv and the device forms: the README's az_move"""

    def __init__(self, n, lists, net, fmt):
        self.env = GoEnv.create(len(lists), board_size=n, device=DEV, features=None)
        self.env.board.replay(lists)
        self.mc = MctsBatch(self.env.board, feature_format=fmt, **OPTS)
        self.net = net
        self.move = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.nr = torch.zeros(len(lists), dtype=torch.uint8, device="cuda")
        self.nr[:NEVER_RESIGN] = 1
        self.active = torch.ones(len(lists), dtype=torch.uint8, device="cuda")

    def az_move(self):
        mc, env = self.mc, self.env
        mc.search_dev(self.net, self.move, self.active)
        a, v = mc.choose_dev(CUTOFF, THRES, seed=self.move ^ SEED, never_resign=self.nr)
        self.res = mc.results_dev()
        obs = env.step(a)
        resigned = a == -1
        ended = obs["done"].bool() | resigned  # read before reset(), which clears done
        env.reset(resigned)
        mc.advance_dev(a)
        mc.reset_dev(ended)
        self.move.add_(1)
        self.a, self.v = a, v


def assert_same(x, y, what):
    if isinstance(x, dict):
        for k in x:
            assert_same(x[k], y[k], f"{what} {k}")
    elif isinstance(x, tuple):
        for i, (a, b) in enumerate(zip(x, y)):
            assert_same(a, b, f"{what} [{i}]")
    else:
        y = y.cpu().numpy() if isinstance(y, torch.Tensor) else y
        assert x.tobytes() == y.tobytes(), what


def run(n, G, moves, fmt, graph, seed):
    """the two loops move for move; with `graph`, move 0 is the warm-up and every later move a replay of one
    captured az_move"""
    lists = openings(n, G, seed)
    net = PlaneNet(n, "cuda", batchsize=0)
    host, dev = Host(n, lists, net, fmt), Device(n, lists, net, fmt)
    ev = dict(noised=0, sampled=0, resigned=0, ended=0, inactive=0)
    g = None
    for k in range(moves):
        active = np.ones(G, np.uint8)
        if k % 3 == 2:
            active[-5:] = 0
        dev.active.copy_(torch.from_numpy(active))
        h = host.move(active)
        if graph and k == 1:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                dev.az_move()
        if g is not None:
            g.replay()
        else:
            dev.az_move()
        torch.cuda.synchronize()
        label = f"move {k}, n={n} {fmt} graph={graph}"
        assert_same(h["actions"], dev.a, f"actions, {label}")
        assert_same(h["values"], dev.v, f"values, {label}")
        assert_same({key: h[key] for key in dev.res}, dev.res, f"results, {label}")
        assert_same(h["after"], after_move(dev.mc, dev.env.board), f"after the move, {label}")
        for key in ("noised", "sampled", "ended"):
            ev[key] += h[key]
        ev["resigned"] += int((h["actions"] == -1).sum())
        ev["inactive"] += int((h["actions"] == -2).sum())
    assert int(net.bad) == 0
    e = host.mc.errors()
    assert e[0] == 0 and e[1] == 0 and e[2] == 0, e
    ev["pruned"] = int(e[3])
    for key in ev:
        assert ev[key] > 0, (key, ev)
    print(f"\n[search_dev] n={n} G={G} {fmt} graph={graph}: {ev}")


@pytest.mark.parametrize("n,G", [(19, 512), (9, 2048)])
def test_a_eager_device_forms_equal_host_loop(n, G):
    run(n, G, 12, "f32", graph=False, seed=n)


@pytest.mark.parametrize("fmt", ["f32", "f16"])
def test_b_captured_move_equals_host_loop(fmt):
    run(9, 2048, 12, fmt, graph=True, seed=3)


def test_c_replays_draw_from_the_device_counters():
    """two consecutive replays of a captured move from identical boards and trees give different noisy root priors
    in at least 99 % of the games; the same replay with the move counter set back gives the same priors, bit for bit"""
    n, G = 9, 2048
    lists = openings(n, G, 7)
    net = PlaneNet(n, "cuda", batchsize=0)
    dev = Device(n, lists, net, "f32")
    dev.nr.fill_(1)
    dev.az_move()  # persistent roots with edges: the noise applies to them at the next begin_move
    saved_gb = GoBatch(G, board_size=n, device=DEV)
    saved_mc = MctsBatch(saved_gb, **OPTS)
    every = torch.arange(G, dtype=torch.int32, device="cuda")
    saved_gb.gather(dev.env.board, every)
    MctsBatch.gather(saved_mc, dev.mc, every)

    def restore():
        dev.env.board.gather(saved_gb, every)
        MctsBatch.gather(dev.mc, saved_mc, every)

    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        dev.mc.search_dev(net, dev.move)
        dev.move.add_(1)
    k = int(dev.move.item())
    priors = []
    for m in (k, k + 1, k):
        restore()
        dev.move.fill_(m)
        g.replay()
        torch.cuda.synchronize()
        assert int(dev.move.item()) == m + 1
        priors.append(dev.mc.root_priors())
    has = (priors[0] >= 0).any(1)
    assert has.mean() > 0.99, has.mean()
    differ = (priors[0] != priors[1]).any(1)
    assert differ[has].mean() >= 0.99, differ[has].mean()
    assert priors[0].tobytes() == priors[2].tobytes()
    assert dev.mc.errors()[0] == 0
