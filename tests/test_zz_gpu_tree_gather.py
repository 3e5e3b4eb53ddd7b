"""Copying search trees between handles on the H100 (MctsBatch.gather, k_gather_trees), at full size.

Scenario: 16 seeded random opening plies, three searched moves chosen on the device (choose with
policy_distri_cutoff 0: the most visited move) and advanced into, then the copy, then more search.  The network
is tests/planenet.py's plane-digest net, a pure function of the leaf planes, so a wrong plane changes priors.
Waves of 8, virtual loss 1, c_puct 1.5, persistent trees, no root noise, rotation_flip 0.

A  2048 19x19 games at 800 rollouts and 8192 9x9 games at 400, on two handles: the destination (trees of its
   own) receives a random permutation with -1 entries; every copied game equals its source right after the copy
   and after one more move on both handles (visits, root value, best_q, total visits, chosen move, tree
   usage), every untouched game is unchanged by the copy.
B  the device form captured in one CUDA graph together with GoBatch.gather and replayed equals the host form,
   and both search on equally.
C  lookahead at scale: 512 19x19 roots x K = 8 branches at 400 rollouts; on 32 sampled roots each branch equals
   a control that rebuilt the root from its moves, played the candidate, advanced and searched; the best
   branch copied back into the roots searches on as the branch does.

Each test prints its wall time, the node pools' peak device memory and torch's max_memory_allocated, with the
card's name and power limit read in the same run."""
import gc
import subprocess
import time

import numpy as np
import pytest
import torch

from tests import planenet
from tests.search_scale import OPENING_PLIES, random_opening

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

DEV = torch.device("cuda", 0)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown card"


class Report:
    """wall time and peak device memory of a test (the node pools are not torch allocations: the lowest free
    memory seen is sampled after every searched move)"""

    def __init__(self, name):
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        self.name, self.t0, self.low = name, time.perf_counter(), None
        self.free0, self.total = torch.cuda.mem_get_info()

    def sample(self):
        torch.cuda.synchronize()
        free, _ = torch.cuda.mem_get_info()
        self.low = free if self.low is None else min(self.low, free)

    def done(self):
        self.sample()
        print(f"\n[{self.name}] {time.perf_counter() - self.t0:.1f} s wall; peak device memory in use "
              f"{(self.total - self.low) / 1e9:.1f} GB of {self.total / 1e9:.1f} GB; torch max_memory_allocated "
              f"{torch.cuda.max_memory_allocated() / 1e9:.2f} GB; {card()}", flush=True)


def opts(R):
    return dict(num_rollouts=R, num_rollouts_per_batch=8, virtual_loss=1, persistent_tree=1, c_puct=1.5, rotation_flip=0)


def new_search(gb, R):
    import elf_b200

    return elf_b200.MctsBatch(gb, **opts(R))


def searched_moves(gb, mc, net, moves, rep=None):
    """`moves` searched moves, each chosen on the device and advanced into; returns the moves played"""
    played = []
    for _ in range(moves):
        mc.search(net)
        if rep:
            rep.sample()
        a, _ = mc.choose(0, 0.0)
        gb.forward(a)
        mc.advance(a)
        played.append(a)
    return played


def build(n, G, R, net, seed, moves=3, rep=None):
    """a GoBatch after the opening and `moves` searched moves, its search handle, and every move played"""
    import elf_b200

    gb = elf_b200.GoBatch(G, board_size=n)
    opening = random_opening([gb], OPENING_PLIES, np.random.default_rng(seed))
    mc = new_search(gb, R)
    return gb, mc, list(opening) + searched_moves(gb, mc, net, moves, rep)


def tables(mc):
    r = mc.results()
    r["priors"] = mc.root_priors()
    r["nodes"], r["edges"] = mc.tree_usage()
    return r


KEYS = ("visits", "priors", "root_value", "best_q", "total_visits", "best_action", "nodes", "edges")


def assert_rows(a, ia, b, ib, label, keys=KEYS):
    """rows ia of the tables a equal rows ib of b, bitwise"""
    for k in keys:
        x, y = np.ascontiguousarray(a[k][ia]), np.ascontiguousarray(b[k][ib])
        if x.tobytes() != y.tobytes():
            bad = np.flatnonzero((x != y).reshape(len(ia), -1).any(1))
            raise AssertionError(f"{label}: {k} differs in {len(bad)} games, e.g. {np.asarray(ia)[bad[:5]]}")


def permutation_with_holes(G_dst, G_src, rng):
    idx = rng.permutation(G_src)[:G_dst].astype(np.int32)
    idx[rng.random(G_dst) < 0.125] = -1
    return idx


@pytest.mark.parametrize("n,G,R", [(19, 2048, 800), (9, 8192, 400)])
def test_a_copies_equal_their_sources(n, G, R):
    rep = Report(f"A {n}x{n} {G} games {R} rollouts")
    net = planenet.PlaneNet(n, "cuda", batchsize=0)
    src, sm, _ = build(n, G, R, net, seed=n, rep=rep)
    dst, dm, _ = build(n, G, R, net, seed=n + 1, moves=1, rep=rep)
    before = tables(dm)
    idx = permutation_with_holes(G, G, np.random.default_rng(7))
    cp, un = np.flatnonzero(idx >= 0), np.flatnonzero(idx < 0)
    dst.gather(src, idx)
    dm.gather(sm, idx)
    assert (dst.getHashCode()[cp] == src.getHashCode()[idx[cp]]).all()
    s0, d0 = tables(sm), tables(dm)
    assert_rows(d0, cp, s0, idx[cp], "copies after the copy")
    assert_rows(d0, un, before, un, "untouched games after the copy")
    for mc in (sm, dm):
        mc.search(net)
        rep.sample()
    s1, d1 = tables(sm), tables(dm)
    assert_rows(d1, cp, s1, idx[cp], "copies after one more move")
    (a_s, v_s), (a_d, v_d) = sm.choose(0, 0.0), dm.choose(0, 0.0)
    assert (a_d[cp] == a_s[idx[cp]]).all() and v_d[cp].tobytes() == v_s[idx[cp]].tobytes()
    assert (s1["total_visits"] >= R).all()
    for mc in (sm, dm):
        assert (mc.errors()[:3] == 0).all(), mc.errors()
    planenet_clean(net)
    rep.done()
    for x in (sm, dm, src, dst):
        x.close()


def planenet_clean(net):
    assert int(net.bad.item()) == 0 and net.calls > 0


def test_b_graph_of_board_and_tree_copies_equals_host_form():
    n, G, R = 9, 1024, 400
    rep = Report(f"B {n}x{n} {G} games {R} rollouts")
    net = planenet.PlaneNet(n, "cuda", batchsize=0)
    src, sm, _ = build(n, G, R, net, seed=3, rep=rep)
    pairs = [build(n, G, R, net, seed=4, moves=1, rep=rep)[:2] for _ in range(2)]
    idx = permutation_with_holes(G, G, np.random.default_rng(8))
    (dh, mh), (dg, mg) = pairs
    dh.gather(src, idx)
    mh.gather(sm, idx)
    it = torch.from_numpy(idx).to(DEV)
    none = torch.full((G,), -1, dtype=torch.int32, device=DEV)
    dg.gather(src, none)  # creates the copies' events outside the capture; copies nothing
    mg.gather(sm, none)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        dg.gather(src, it)
        mg.gather(sm, it)
    graph.replay()
    torch.cuda.synchronize()
    assert (dg.getHashCode() == dh.getHashCode()).all()
    all_g = np.arange(G)
    assert_rows(tables(mg), all_g, tables(mh), all_g, "graph replay vs host form")
    for mc in (mh, mg):
        mc.search(net)
        rep.sample()
    assert_rows(tables(mg), all_g, tables(mh), all_g, "one more move")
    planenet_clean(net)
    rep.done()
    for x in (sm, mh, mg, src, dh, dg):
        x.close()


def test_c_lookahead_at_scale():
    import elf_b200

    n, G, K, R, S = 19, 512, 8, 400, 32
    rep = Report(f"C {n}x{n} {G} roots x {K} branches {R} rollouts")
    net = planenet.PlaneNet(n, "cuda", batchsize=0)
    roots, rm, moves = build(n, G, R, net, seed=5, rep=rep)
    rm.search(net)
    r0 = tables(rm)
    cand = np.argsort(-r0["visits"], axis=1, kind="stable")[:, :K].astype(np.int32)  # [G, K]
    assert (np.take_along_axis(r0["visits"], cand, 1) >= 0).all()  # root edges: legal moves
    to_b = torch.arange(G, dtype=torch.int32, device=DEV).repeat_interleave(K)
    br = elf_b200.GoBatch(G * K, board_size=n)
    bm = new_search(br, R)
    br.gather(roots, to_b)
    bm.gather(rm, to_b)
    assert br.forward(cand.reshape(-1)).all()
    bm.advance(cand.reshape(-1))
    bm.search(net)
    rep.sample()
    rb = tables(bm)
    # controls: the sampled roots rebuilt from their moves (a game's search depends on nothing but its own
    # position and tree), K slots each, the candidate played and advanced, then searched
    sample = np.sort(np.random.default_rng(9).choice(G, S, replace=False))
    rows = np.repeat(sample, K)
    cg = elf_b200.GoBatch(S * K, board_size=n)
    for a in moves[:OPENING_PLIES]:
        assert cg.forward(a[rows]).all()
    cm = new_search(cg, R)
    for a in moves[OPENING_PLIES:]:
        cm.search(net)
        got, _ = cm.choose(0, 0.0)
        assert (got == a[rows]).all()
        cg.forward(got)
        cm.advance(got)
    cm.search(net)
    ck = cand[sample].reshape(-1)
    assert cg.forward(ck).all()
    cm.advance(ck)
    cm.search(net)
    bsel = (rows * K + np.tile(np.arange(K), S)).astype(np.int64)
    assert_rows(tables(cm), np.arange(S * K), rb, bsel, "branches vs controls")
    # the best branch back into the roots
    best = (np.arange(G) * K + rb["best_q"].reshape(G, K).argmax(1)).astype(np.int32)
    roots.gather(br, best)
    rm.gather(bm, best)
    for mc in (rm, bm):
        mc.search(net)
        rep.sample()
    assert_rows(tables(rm), np.arange(G), tables(bm), best, "roots after copying back the best branch")
    for mc in (rm, bm, cm):
        assert (mc.errors()[:3] == 0).all(), mc.errors()
    planenet_clean(net)
    rep.done()
    for x in (rm, bm, cm, roots, br, cg):
        x.close()
