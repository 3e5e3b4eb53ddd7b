"""Copying search trees between handles (elfb200_mcts_gather / elfb200_mcts_gather_dev, k_gather_trees,
MctsBatch.gather): a copied tree is bitwise indistinguishable from its source under continued search.

CPU: the kernels run on the SIMT emulator build of the kernel sources (tests/simt_emu), under every lane order.
The network is oracles.fakenet keyed by the leaf hash, with rotation_flip = 0 and no root noise, so a search is
a pure function of the board and the tree.  The emulator's search class has no gather method of its own: the
product's MctsBatch.gather / tree_usage are called on it (they only use the handle and the library).
tests/test_zz_gpu_tree_gather.py runs the checks at full size on an H100."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from elf_b200.mcts import MctsBatch
from tests import oracles
from tests.test_gather import ko_moves, superko_opening
from tests.test_handicap import SEARCH_OPTS

pytestmark = pytest.mark.timeout(900)

ERR_ARG = -1  # ELFB200_ERR_ARG (include/elfb200.h)
R = SEARCH_OPTS["num_rollouts"]  # rollouts per move (whole waves of 8)


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


# ---- scenario pieces ----------------------------------------------------------------------------------
def random_plies(gb, rng, plies, games):
    """`plies` uniform legal moves (a pass when no point is legal) in each of `games`; the others stay"""
    n = gb.board_size
    for _ in range(plies):
        lg = gb.legal_mask()
        a = np.full(gb.num_games, -1, np.int32)
        for g in games:
            c = np.flatnonzero(lg[g, :-1])
            a[g] = int(rng.choice(c)) if len(c) else n * n
        assert gb.forward(a)[list(games)].all()


def make_sources(emu, n, rng):
    """source positions as in tests/test_gather.py's search on copies: on 9x9 (G = 7, one partial warp of
    the per-game kernels) the superko opening, a ko fight, handicap stones, random plies and a fresh game; on
    19x19 (G = 4) a ko fight, handicap stones and random plies"""
    if n == 9:
        G, lists, hcap, rand = 7, {0: superko_opening(), 1: ko_moves(n)}, {2: [20, 60, 24], 6: [20, 60]}, {3: 30, 4: 12, 6: 8}
    else:
        G, lists, hcap, rand = 4, {0: ko_moves(n)}, {1: [60, 300, 72, 288]}, {2: 40, 3: 10, 1: 6}
    gb = emu.emu_batch(G, n)
    for t in range(max(len(m) for m in lists.values())):
        gb.forward(np.array([lists[g][t] if g in lists and t < len(lists[g]) else -1 for g in range(G)], np.int32))
    assert all(ok.all() for ok in gb.place_handicap([hcap.get(g, []) for g in range(G)]))
    for g, k in rand.items():
        random_plies(gb, rng, k, [g])
    return gb


def search_move(mc):
    """one searched move: the root tables, priors and the planes of every leaf evaluated, per game in
    evaluation order as (leaf hash, planes)"""
    P1 = mc.gb.num_actions
    leaves = {}

    def actor(batch):
        h, g, _ = mc.leaf_info()
        s = batch["s"].numpy()
        for i, (hh, gg) in enumerate(zip(h, g)):
            leaves.setdefault(int(gg), []).append((int(hh), s[i].copy()))
        pi, v = oracles.fakenet(h, P1)
        return {"pi": torch.from_numpy(pi), "V": torch.from_numpy(v)}

    res = mc.act(actor)
    res["priors"] = mc.root_priors()
    res["leaves"] = leaves
    res["usage"] = MctsBatch.tree_usage(mc)
    return res


def play(gb, mc, actions):
    """play the chosen moves (-1: the game has no move) and keep their subtrees"""
    a = np.asarray(actions, np.int32)
    ok = gb.forward(a)
    assert ok[a >= 0].all()
    mc.advance(a)


def assert_same_game(a, i, b, j, label):
    """game i of the search results `a` is bitwise game j of `b`"""
    for k in ("visits", "priors"):
        np.testing.assert_array_equal(a[k][i].view(np.int32), b[k][j].view(np.int32), err_msg=f"{k} {label}")
    for k in ("root_value", "best_q", "total_visits", "best_action"):
        assert a[k][i].tobytes() == b[k][j].tobytes(), f"{k} {label}: {a[k][i]} vs {b[k][j]}"
    for k in (0, 1):
        assert a["usage"][k][i] == b["usage"][k][j], f"tree usage {label}"
    la, lb = a["leaves"].get(i, []), b["leaves"].get(j, [])
    assert [h for h, _ in la] == [h for h, _ in lb], f"leaf hashes {label}"
    for (h, pa), (_, pb) in zip(la, lb):
        np.testing.assert_array_equal(pa, pb, err_msg=f"leaf planes {label} {h:x}")


def run_replica_continuation(emu, n, seed, opts, pressure=False):
    """Sources with two searched moves on persistent trees; a destination with trees of its own, and a control
    handle that runs the destination's moves but never receives the copy.  Index with duplicates, -1, G_src
    and int32's extremes (or, with `pressure`, a permutation of the sources, so that whole handles compare).
    Then one more searched move on all three, advance, and another: every copied game equals its source
    (visit tables, priors, root value, best_q, total visits, best action, tree usage, the planes of every
    leaf), every untouched game equals the control.  Returns the prune counters' advance (src, dst)."""
    rng = np.random.default_rng(seed)
    src = make_sources(emu, n, rng)
    Gs = src.num_games
    sm = emu.EmuSearch(src, rotation_flip=0, **opts)
    for _ in range(2):
        play(src, sm, search_move(sm)["best_action"])
    if pressure:
        idx = rng.permutation(Gs).astype(np.int32)
    else:
        idx = np.concatenate([[Gs - 1, Gs - 1, -1, Gs, -(2 ** 31), 2 ** 31 - 1], rng.permutation(Gs)]).astype(np.int32)
    Gd = len(idx)
    pair = []
    for _ in range(2):  # destination and control: the same moves, the same trees
        gb = emu.emu_batch(Gd, n)
        random_plies(gb, np.random.default_rng(seed + 1), 6, range(Gd))
        mc = emu.EmuSearch(gb, rotation_flip=0, **opts)
        play(gb, mc, search_move(mc)["best_action"])
        pair.append((gb, mc))
    (dst, dm), (ctl, cm) = pair
    dst.gather(src, idx)
    MctsBatch.gather(dm, sm, idx)
    copied = [(i, int(s)) for i, s in enumerate(idx) if 0 <= s < Gs]
    untouched = [i for i, s in enumerate(idx) if not 0 <= s < Gs]
    assert len(copied) == Gs + (0 if pressure else 2)
    e0 = (sm.errors()[3], dm.errors()[3])
    for move in range(2):
        rs, rd, rc = search_move(sm), search_move(dm), search_move(cm)
        for i, s in copied:
            assert_same_game(rd, i, rs, s, f"copy {i} of {s}, move {move}")
        for i in untouched:
            assert_same_game(rd, i, rc, i, f"untouched {i}, move {move}")
        for gb, mc, r in ((src, sm, rs), (dst, dm, rd), (ctl, cm, rc)):
            play(gb, mc, r["best_action"])
    for mc in (sm, dm, cm):
        e = mc.errors()
        assert e[0] == 0 and e[1] == 0 and e[2] == 0, e
    grown = (int(sm.errors()[3] - e0[0]), int(dm.errors()[3] - e0[1]))
    for x in (sm, dm, cm, src, dst, ctl):
        x.close()
    return grown


def build_roots(emu):
    """R = 3 9x9 roots (a ko fight, random plies, handicap stones) with two searched moves played and a third
    search on the position reached; deterministic, so every call builds the same boards and trees"""
    n = 9
    gb = emu.emu_batch(3, n)
    km = ko_moves(n)
    for a in km:
        gb.forward(np.array([a, -1, -1], np.int32))
    random_plies(gb, np.random.default_rng(11), 20, [1])
    gb.place_handicap([[], [], [20, 60, 24]])
    mc = emu.EmuSearch(gb, rotation_flip=0, **SEARCH_OPTS)
    for _ in range(2):
        play(gb, mc, search_move(mc)["best_action"])
    return gb, mc, search_move(mc)


def run_lookahead(emu, K=4):
    """One-ply lookahead that keeps the root's search: copy boards and trees into K branch slots per root,
    play K distinct candidates (the root's most visited edges), advance every branch into its candidate's
    subtree and search.  Each branch equals a control built from scratch: the same root, the candidate played
    and advanced, and searched.  Then the best branch is copied back into the root handle and both search once
    more: the roots equal their branches."""
    roots, rm, r0 = build_roots(emu)
    Rn = roots.num_games
    cand = np.argsort(-r0["visits"], axis=1, kind="stable")[:, :K].astype(np.int32)  # [R, K]
    assert (np.take_along_axis(r0["visits"], cand, 1) > 0).all()
    to_branches = np.repeat(np.arange(Rn), K).astype(np.int32)
    br = emu.emu_batch(Rn * K, 9)
    bm = emu.EmuSearch(br, rotation_flip=0, **SEARCH_OPTS)
    br.gather(roots, to_branches)
    MctsBatch.gather(bm, rm, to_branches)
    play(br, bm, cand.reshape(-1))
    rb = search_move(bm)
    for k in range(K):
        cg, cm, _ = build_roots(emu)
        play(cg, cm, cand[:, k])
        rc = search_move(cm)
        for r in range(Rn):
            assert_same_game(rb, r * K + k, rc, r, f"branch {k} of root {r}")
        cm.close()
        cg.close()
    best = (np.arange(Rn) * K + rb["best_q"].reshape(Rn, K).argmax(1)).astype(np.int32)
    roots.gather(br, best)
    MctsBatch.gather(rm, bm, best)
    rr, rb2 = search_move(rm), search_move(bm)
    for r in range(Rn):
        assert_same_game(rr, r, rb2, int(best[r]), f"root {r} after copying back branch {best[r]}")
    for x in (rm, bm, roots, br):
        x.close()


@pytest.mark.parametrize("n", [9, 19])
def test_replica_continues_as_its_source(emu, lane_order, n):
    run_replica_continuation(emu, n, seed=n, opts=SEARCH_OPTS)


def test_replica_under_pool_pressure(emu, lane_order):
    """a node pool of rollouts + 8 slots per game: a persistent tree is pruned whenever the subtree kept by
    advance holds more than 7 nodes (with rollouts + 64 it never does at 64 rollouts); the copies still
    continue as their sources, and both handles count the same number of prunes"""
    grown = run_replica_continuation(emu, 9, seed=5, opts=dict(SEARCH_OPTS, nodes_per_game=R + 8), pressure=True)
    assert grown[0] == grown[1] >= 7, grown


def test_lookahead_keeps_the_roots_search(emu, lane_order):
    run_lookahead(emu)


def readback(mc):
    """results, priors and tree usage without a search"""
    r = mc.results()
    r["priors"] = mc.root_priors()
    r["usage"] = MctsBatch.tree_usage(mc)
    return r


def assert_same_readback(a, b, label):
    for k in ("visits", "priors", "root_value", "best_q", "total_visits", "best_action"):
        assert a[k].tobytes() == b[k].tobytes(), f"{k} {label}"
    assert all((x == y).all() for x, y in zip(a["usage"], b["usage"])), f"usage {label}"


def refused(L, fn, dst, src, idx, why):
    """fn(dst, src, idx) returns ERR_ARG with `why` in the message and enqueues nothing on either context"""
    ctxs = [m.gb for m in (dst, src) if m is not None]
    n0 = [gb.launch_count() for gb in ctxs]
    assert fn(dst._m if dst is not None else None, src._m if src is not None else None, idx) == ERR_ARG
    assert why.encode() in L.elfb200_last_error(), L.elfb200_last_error()
    assert [gb.launch_count() for gb in ctxs] == n0


def test_tree_gather_arguments(emu):
    """every refused call returns ERR_ARG, enqueues nothing and changes neither handle; two handles on one
    board context may copy"""
    L = emu.emu_lib()
    a, b, c = emu.emu_batch(4, 9), emu.emu_batch(3, 9), emu.emu_batch(4, 19)
    random_plies(a, np.random.default_rng(1), 5, range(4))
    ma, mb = emu.EmuSearch(a, rotation_flip=0, **SEARCH_OPTS), emu.EmuSearch(b, rotation_flip=0, **SEARCH_OPTS)
    mc = emu.EmuSearch(c, rotation_flip=0, **SEARCH_OPTS)
    small = emu.EmuSearch(b, rotation_flip=0, **dict(SEARCH_OPTS, nodes_per_game=2 * R + 100))
    for m in (ma, mb):
        search_move(m)
    before = [readback(m) for m in (ma, mb)]
    idx = np.zeros(4, np.int32).ctypes.data
    for fn in (L.elfb200_mcts_gather, L.elfb200_mcts_gather_dev):
        refused(L, fn, None, mb, idx, "NULL")
        refused(L, fn, ma, None, idx, "NULL")
        refused(L, fn, ma, mb, None, "NULL")
        refused(L, fn, ma, ma, idx, "same search handle")
        refused(L, fn, ma, mc, idx, "board sizes differ")
        refused(L, fn, mc, ma, idx, "board sizes differ")
        refused(L, fn, ma, small, idx, "nodes_per_game differs")
        refused(L, fn, small, mb, idx, "nodes_per_game differs")
    for m, r in zip((ma, mb), before):
        assert_same_readback(readback(m), r, "after the refused calls")
    # a wave open on either side: its claimed leaves and applied virtual loss must not be copied
    mb.begin_move()
    assert mb.select().shape[0] > 0
    open_b = readback(mb)
    for fn in (L.elfb200_mcts_gather, L.elfb200_mcts_gather_dev):
        refused(L, fn, ma, mb, idx, "src handle has a wave open")
        refused(L, fn, mb, ma, idx, "dst handle has a wave open")
    assert_same_readback(readback(ma), before[0], "beside an open wave")
    assert_same_readback(readback(mb), open_b, "with its wave open")
    h, _, _ = mb.leaf_info()
    pi, v = oracles.fakenet(h, mb.gb.num_actions)
    mb.expand_backup(torch.from_numpy(pi), torch.from_numpy(v))
    for _ in range(mb.waves_per_move - 1):  # the rest of the move, so that its tree is whole again
        s = mb.select()
        h, _, _ = mb.leaf_info()
        pi, v = oracles.fakenet(h, mb.gb.num_actions)
        if s.shape[0]:
            mb.expand_backup(torch.from_numpy(pi), torch.from_numpy(v))
        else:
            mb.expand_backup(None, None)
    # two handles on one board context (a tree per colour): after a copy of every game, both search on equally
    m2 = emu.EmuSearch(b, rotation_flip=0, **SEARCH_OPTS)
    MctsBatch.gather(m2, mb, np.arange(3))
    assert_same_readback(readback(m2), readback(mb), "copy on the same context")
    r1, r2 = search_move(mb), search_move(m2)
    for g in range(3):
        assert_same_game(r2, g, r1, g, f"same context {g}")
    with pytest.raises(ValueError):
        MctsBatch.gather(m2, mb, np.arange(4))
    for x in (ma, mb, mc, small, m2, a, b, c):
        x.close()


_ASAN_CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests/simt_emu")
import build
from elf_b200 import lib as _l
from elf_b200.mcts import MctsBatch
from tests import emu as E
E._lib = _l.load_library(build.build(asan=True))
from tests.test_tree_gather import SEARCH_OPTS, make_sources, play, search_move
for n, Gd in ((9, 11), (19, 8)):
    src = make_sources(E, n, np.random.default_rng(n))
    Gs = src.num_games
    sm = E.EmuSearch(src, rotation_flip=0, **SEARCH_OPTS)
    play(src, sm, search_move(sm)["best_action"])
    search_move(sm)
    dst = E.emu_batch(Gd, n)
    dm = E.EmuSearch(dst, rotation_flip=0, **SEARCH_OPTS)
    search_move(dm)
    idx = np.array([Gs, -1, 0, Gs - 1, -(2 ** 31), 2 ** 31 - 1] + [g % Gs for g in range(Gd - 6)], np.int32)
    dst.gather(src, idx)
    MctsBatch.gather(dm, sm, idx)
    _l.check(E._lib, E._lib.elfb200_mcts_gather_dev(dm._m, sm._m, idx.ctypes.data))
    r = search_move(dm)
    assert (r["visits"][2] == search_move(sm)["visits"][0]).all()
    for x in (sm, dm, src, dst):
        x.close()
print("ASAN TREE GATHER CLEAN")
"""


def test_tree_gather_clean_under_address_sanitizer(emu):
    """the tree copy with negative and out-of-range indices, and searches on the copies, on the emulator build
    under AddressSanitizer (every device buffer is a heap allocation there, so any read or write outside a
    node pool is reported)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        asan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        pytest.skip(f"no gcc: {e}")
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("libasan is not installed")
    env = dict(os.environ, LD_PRELOAD=os.path.realpath(asan), ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0")
    r = subprocess.run([sys.executable, "-c", _ASAN_CHILD, root], env=env, capture_output=True, text=True, timeout=850)
    assert r.returncode == 0 and "ASAN TREE GATHER CLEAN" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]
