"""Copying games between batches (elfb200_gather_games / elfb200_gather_games_dev, k_gather, GoBatch.gather,
GoEnv.load) against the compiled reference's GoState copy constructor (ref_clone).

CPU: the kernels run on the SIMT emulator build of the kernel sources (tests/simt_emu), under every lane
order; the GoEnv tensors are CPU tensors there.  tests/test_zz_gpu_gather.py runs the checks at full batch
size on an H100."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import oracles
from tests.test_env import KOMI, assert_obs, end_reason, pick_actions, step_and_check
from tests.test_handicap import SEARCH_OPTS, assert_same_state, need_ref, ref_place_handicap

pytestmark = pytest.mark.timeout(900)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ERR_ARG = -1  # ELFB200_ERR_ARG (include/elfb200.h)

# After the 64-ply opening of the 9x9 "superko in tree" search scenario (mcts_superko_opening_9.json), black
# plays 4 and white recaptures at 3: the position after the recapture repeats an earlier position of the game,
# so the reference ends the game by positional superko.
SUPERKO_REPLY = (4, 3)


def ref_clone(r):
    """GoState's copy constructor of the compiled reference (oracle/ref_shim.cc: ref_clone)"""
    c = oracles.Ref.__new__(oracles.Ref)
    c.L, c.n, c.p = r.L, r.n, r.L.ref_clone(r.p)
    return c


def superko_opening():
    return json.load(open(os.path.join(GOLDEN, "mcts_superko_opening_9.json")))["openings"][0]


def ko_moves(n):
    """black takes a simple ko at (2,1): afterwards white may not retake at (1,1) at once"""
    a = lambda x, y: x * n + y  # noqa: E731
    return [a(1, 0), a(2, 0), a(0, 1), a(3, 1), a(1, 2), a(2, 2), a(6, 6), a(1, 1), a(2, 1)]


def random_moves(r, rng, plies, p_pass=0.0):
    """plays up to `plies` uniform legal moves (a pass when none is legal or with probability p_pass) on the
    reference state `r`; returns them"""
    n = r.n
    out = []
    for _ in range(plies):
        if r.terminated():
            break
        cand = np.flatnonzero(r.legal())
        a = n * n if len(cand) == 0 or rng.random() < p_pass else int(rng.choice(cand))
        assert r.forward(a)
        out.append(a)
    return out


def ply_cap_moves(n):
    """a move list that reaches the 2N^2 ply cap: uniform legal moves (eyes included), a pass only when
    nothing else is legal; the first seed whose game neither passes twice nor repeats a position"""
    for seed in range(200):
        r = oracles.Ref(n)
        mv = random_moves(r, np.random.default_rng(seed), 2 * n * n)
        if r.terminated() and not r.info()[10] and not r.info()[11]:
            return mv
    raise AssertionError("no seed reaches the ply cap")


def make_sources(make_batch, n, rng):
    """a source batch and one reference state per game, in a mix of states: fresh, an active simple ko, a
    handicap position at ply 1, a game ended by two passes, a mid-game position, and on 9x9 also games ended
    by superko and by the ply cap (G = 7 on 9x9: three games per warp, so warps mix copied and untouched
    games; 5 on 19x19)"""
    P = n * n
    refs = [oracles.Ref(n) for _ in range(7 if n == 9 else 5)]
    G = len(refs)
    gb = make_batch(G, n)
    stones = [[] for _ in range(G)]
    stones[2] = [3 * n + 3, 5 * n + 5, 2 * n + 6] if n == 9 else [3 * n + 3, 15 * n + 15, 3 * n + 15, 9 * n + 9]
    ok = gb.place_handicap(stones)
    assert all(ref_place_handicap(refs[2], a) for a in stones[2]) and ok[2].all()
    lists = [[] for _ in range(G)]
    lists[1] = ko_moves(n)
    for a in lists[1]:
        assert refs[1].forward(a)
    lists[3] = random_moves(refs[3], rng, 30) + [P, P]
    assert refs[3].forward(P) and refs[3].forward(P) and refs[3].terminated()
    lists[4] = random_moves(refs[4], rng, 150 if n == 19 else 40, p_pass=0.02)
    if n == 9:
        lists[5] = superko_opening() + list(SUPERKO_REPLY)
        for a in lists[5]:
            refs[5].forward(a)
        lists[6] = ply_cap_moves(n)
        for a in lists[6]:
            assert refs[6].forward(a)
    for t in range(max(len(m) for m in lists)):
        acts = np.array([m[t] if t < len(m) else -1 for m in lists], np.int32)
        gb.forward(acts)
    info = np.array([r.info() for r in refs])
    assert info[1, 6] >= 0  # the ko
    assert info[2, 0] == 1 and info[2, 1] == 2  # the handicap position: ply 1, white to move
    assert [end_reason(refs[g]) for g in range(G) if refs[g].terminated()] == (
        ["two_pass", "superko", "ply_cap"] if n == 9 else ["two_pass"])
    assert_same_state(gb, refs, "sources", full=False)
    return gb, refs


def run_copy_equals_reference(make_batch, n, seed):
    """every copied game equals ref_clone of its source in everything observable (hash, info, stones, legal,
    true eyes, tt score, evaluate, AGZ and DarkForest planes under all 8 D4 codes); destination games with an
    index of -1 or out of range keep their state; the source batch is unchanged.  Destinations larger and
    smaller than the source, indices with duplicates."""
    rng = np.random.default_rng(seed)
    src, srefs = make_sources(make_batch, n, rng)
    G = src.num_games
    for Gd in (G + 4, 4):
        dst = make_batch(Gd, n)
        drefs = [oracles.Ref(n) for _ in range(Gd)]
        for t in range(12):  # the untouched games have a position of their own
            acts = pick_actions(rng, drefs, n, p_pass=0.0)
            np.testing.assert_array_equal(dst.forward(acts), [r.forward(int(a)) if a >= 0 else False
                                                              for r, a in zip(drefs, acts)])
        idx = rng.integers(0, G, Gd).astype(np.int64)
        idx[0] = idx[1] = G - 1  # a duplicate
        idx[2] = -1
        idx[3] = G if Gd > G else 10 ** 9  # out of range
        if Gd > G:
            idx[4], idx[5] = -7, -(2 ** 40)
            idx[6:] = rng.permutation(G)[: Gd - 6]
        dst.gather(src, idx)
        for i, s in enumerate(idx):
            if 0 <= s < G:
                drefs[i] = ref_clone(srefs[s])
        assert_same_state(dst, drefs, f"after the copy into {Gd} games")
        assert_same_state(src, srefs, "the source after the copy")
        dst.close()
    src.close()


def run_copies_played_on(make_env, n, seed):
    """source and copies are stepped independently through GoEnv.step with different random actions, each
    against its own cloned reference, until every destination game has ended at least once: ok, done, value
    bit for bit, legal, info and hash every ply"""
    from elf_b200.env import GoEnv

    rng = np.random.default_rng(seed)
    src, srefs = make_sources(make_env.batch, n, rng)
    G = src.num_games
    idx = np.concatenate([np.arange(G), rng.integers(0, G, 3), [-1]]).astype(np.int32)
    dst = make_env(len(idx), n)
    dst.board.gather(src, idx)
    drefs = [ref_clone(srefs[s]) if s >= 0 else oracles.Ref(n) for s in idx]
    senv = GoEnv(src, device=dst.device)
    assert_obs(dst, dst.observe(), drefs, "after the copy")
    finished = np.zeros(len(idx), int)
    t = 0
    while finished.min() < 1:
        step_and_check(senv, srefs, pick_actions(rng, srefs, n), None, f"source ply {t}")
        obs, done, _ = step_and_check(dst, drefs, pick_actions(rng, drefs, n), None, f"copy ply {t}")
        assert_obs(dst, obs, drefs, f"copy ply {t}")
        assert_obs(senv, senv.obs, srefs, f"source ply {t}")
        finished += done
        t += 1
        assert t < 20 * n * n
    dst.close()
    src.close()


def run_superko_record_copied(make_env):
    """the copied superko record is the destination's own: the source game is reset between the copy and
    the moves, and the destination still ends by positional superko on the reference's ply with its value;
    copied after the first of the two moves, the record holds that move's entry too"""
    n = 9
    opening = superko_opening()
    probe = oracles.Ref(n)
    for a in opening:
        probe.forward(a)
    c = ref_clone(probe)
    assert c.forward(SUPERKO_REPLY[0]) and c.forward(SUPERKO_REPLY[1])
    assert c.terminated() and end_reason(c) == "superko"
    for split in (0, 1):  # moves of the reply played before the copy
        src = make_env.batch(2, n)
        sref = oracles.Ref(n)
        pre = opening + list(SUPERKO_REPLY[:split])
        for a in pre:
            sref.forward(a)
            src.forward(np.array([a, -1], np.int32))
        dst = make_env(3, n)
        dst.reset()
        dst.board.gather(src, np.array([-1, 0, -1], np.int32))
        src.reset()
        assert int(src.getHashCode()[0]) == 0
        refs = [oracles.Ref(n), ref_clone(sref), oracles.Ref(n)]
        for t, a in enumerate(SUPERKO_REPLY[split:]):
            last = t == len(SUPERKO_REPLY) - split - 1
            _, done, reasons = step_and_check(dst, refs, np.array([-1, a, -1], np.int32), None, f"reply {t}")
            assert done.tolist() == [False, last, False]
        assert reasons == ["superko"]
        assert dst.value[1].item() == np.float32(c.evaluate(KOMI)) == 1.0
        dst.close()
        src.close()


def run_search_on_copies(make_batch, make_search, n=9):
    """MctsBatch (fake network keyed by the leaf hash, 64 rollouts) on copied positions equals the search on
    the originals: root visits, priors, chosen moves, and the planes of every leaf.  The sources include the
    superko opening, whose tree holds a recapture that repeats a position of the game."""
    rng = np.random.default_rng(3)
    P1 = n * n + 1
    src = make_batch(4, n)
    lists = [superko_opening(), ko_moves(n), [], random_moves(oracles.Ref(n), rng, 30)]
    for t in range(max(len(m) for m in lists)):
        src.forward(np.array([m[t] if t < len(m) else -1 for m in lists], np.int32))
    src.place_handicap([[], [], [20, 60, 24], []])
    idx = np.array([2, 0, 3, 1, 0], np.int32)
    dst = make_batch(len(idx), n)
    dst.forward(np.array([40] * len(idx), np.int32))  # a position of their own before the copy
    dst.gather(src, idx)
    out = {}
    for name, gb in (("src", src), ("dst", dst)):
        mc = make_search(gb, rotation_flip=0, **SEARCH_OPTS)
        leaves = {}  # (game, leaf hash) -> the planes of its evaluations, in order

        def actor(batch, mc=mc, leaves=leaves):
            h, g, _ = mc.leaf_info()
            s = batch["s"].cpu().numpy()
            for i, (hh, gg) in enumerate(zip(h, g)):
                leaves.setdefault((int(gg), int(hh)), []).append(s[i].copy())
            pi, v = oracles.fakenet(h, P1)
            return {"pi": torch.from_numpy(pi).to(mc.device), "V": torch.from_numpy(v).to(mc.device)}

        res = mc.act(actor)
        out[name] = (res, mc.root_priors(), leaves)
        assert (mc.errors() == 0).all()
        mc.close()
    (rs, ps, ls), (rd, pd, ld) = out["src"], out["dst"]
    for i, s in enumerate(idx):
        np.testing.assert_array_equal(rd["visits"][i], rs["visits"][s], err_msg=f"visits {i}")
        np.testing.assert_array_equal(pd[i], ps[s], err_msg=f"priors {i}")
        assert rd["best_action"][i] == rs["best_action"][s] and rd["total_visits"][i] == rs["total_visits"][s]
        mine = {h: v for (g, h), v in ld.items() if g == i}
        theirs = {h: v for (g, h), v in ls.items() if g == s}
        assert len(mine) > 10 and mine.keys() == theirs.keys(), f"leaves {i}"
        for h in mine:
            np.testing.assert_array_equal(np.array(mine[h]), np.array(theirs[h]), err_msg=f"leaf planes {i} {h:x}")
    dst.close()
    src.close()


def run_env_load(make_env, n=9):
    """GoEnv.load: the observation equals observe on the same positions (legal, info, AGZ planes); ok /
    done / value of the loaded games are cleared and the others' kept; a GoEnv source works as a GoBatch"""
    rng = np.random.default_rng(9)
    src, srefs = make_sources(make_env.batch, n, rng)
    G = src.num_games
    env = make_env(6, n, features="f32")
    refs = [oracles.Ref(n) for _ in range(6)]
    env.reset()
    for t in range(10):
        step_and_check(env, refs, pick_actions(rng, refs, n, p_pass=0.0), None, f"ply {t}")
    env.ok.fill_(1)
    env.done.fill_(1)
    env.value.fill_(0.5)
    idx = np.array([5, -1, 1, G, 2, 0], np.int32)
    d4 = rng.integers(0, 8, 6).astype(np.int32)
    obs = env.load(src, torch.from_numpy(idx).to(env.device), torch.from_numpy(d4).to(env.device))
    loaded = (idx >= 0) & (idx < G)
    assert obs["ok"].tolist() == (~loaded).astype(int).tolist() and obs["done"].tolist() == obs["ok"].tolist()
    assert obs["value"].tolist() == np.where(loaded, 0.0, 0.5).tolist()
    refs = [ref_clone(srefs[s]) if m else r for s, m, r in zip(idx, loaded, refs)]
    assert_obs(env, obs, refs, "after the load")
    got = {k: obs[k].clone() for k in ("legal", "info", "planes")}
    again = env.observe(torch.from_numpy(d4).to(env.device))
    for k, v in got.items():
        assert torch.equal(v, again[k]), k
    planes = obs["planes"].cpu().numpy()
    for g, r in enumerate(refs):
        np.testing.assert_array_equal(planes[g], r.features(int(d4[g])), err_msg=f"AGZ g={g}")
    # a GoEnv as the source
    from elf_b200.env import GoEnv

    senv = GoEnv(src, device=env.device)
    obs = env.load(senv, torch.tensor([0, 0, -1, -1, -1, 4], dtype=torch.int32, device=env.device))
    refs[0], refs[1], refs[5] = ref_clone(srefs[0]), ref_clone(srefs[0]), ref_clone(srefs[4])
    assert_obs(env, obs, refs, "GoEnv source")
    with pytest.raises(ValueError):
        env.load(src, torch.zeros(6, dtype=torch.int64, device=env.device))
    env.close()
    src.close()


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


@pytest.fixture
def make_env(emu):
    from elf_b200.env import GoEnv

    def make(G, n, **kw):
        return GoEnv(emu.emu_batch(G, n), device="cpu", **kw)

    make.batch = emu.emu_batch
    return make


@pytest.mark.parametrize("n", [9, 19])
def test_copy_equals_reference_copy(emu, lane_order, n):
    need_ref(n)
    run_copy_equals_reference(emu.emu_batch, n, seed=n)


@pytest.mark.parametrize("n", [9, 19])
def test_copies_stay_equal_when_played_on(make_env, lane_order, n):
    need_ref(n)
    run_copies_played_on(make_env, n, seed=2 * n)


def test_copied_superko_record(make_env, lane_order):
    need_ref(9)
    run_superko_record_copied(make_env)


def test_search_on_copies_equals_search_on_originals(emu, lane_order):
    need_ref(9)
    run_search_on_copies(emu.emu_batch, emu.EmuSearch)


def test_env_load(make_env, lane_order):
    need_ref(9)
    run_env_load(make_env)


def test_gather_arguments(emu):
    L = emu.emu_lib()
    a, b, c = emu.emu_batch(4, 9), emu.emu_batch(3, 9), emu.emu_batch(4, 19)
    a.forward(np.array([40, 41, 42, 43], np.int32))
    before = a.getHashCode()
    idx = np.zeros(4, np.int32)
    for fn in (L.elfb200_gather_games, L.elfb200_gather_games_dev):
        assert fn(None, b._ctx, idx.ctypes.data) == ERR_ARG
        assert fn(a._ctx, None, idx.ctypes.data) == ERR_ARG
        assert fn(a._ctx, b._ctx, None) == ERR_ARG
        assert fn(a._ctx, a._ctx, idx.ctypes.data) == ERR_ARG
        assert b"same context" in L.elfb200_last_error()
        assert fn(a._ctx, c._ctx, idx.ctypes.data) == ERR_ARG and fn(c._ctx, a._ctx, idx.ctypes.data) == ERR_ARG
        assert b"board sizes differ" in L.elfb200_last_error()
    assert (a.getHashCode() == before).all() and (c.getHashCode() == 0).all()
    n0 = a.launch_count()
    idx = np.array([-1, 5, 2, -3], np.int32)
    assert fn(a._ctx, b._ctx, idx.ctypes.data) == 0  # the _dev form
    assert a.launch_count() == n0 + 1
    assert (a.getHashCode() == np.array([before[0], before[1], 0, before[3]])).all()
    for x in (a, b, c):
        x.close()


_ASAN_CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests/simt_emu")
import build
from elf_b200 import lib as _l
from tests import emu as E
E._lib = _l.load_library(build.build(asan=True))
for n, Gs, Gd in ((9, 7, 11), (19, 3, 8)):
    src, dst = E.emu_batch(Gs, n), E.emu_batch(Gd, n)
    rng = np.random.default_rng(n)
    src.replay([[int(a) for a in rng.integers(0, n * n + 1, int(rng.integers(0, 2 * n * n)))] for _ in range(Gs)])
    idx = np.array([Gs, -1, 0, Gs - 1, -(2 ** 31), 2 ** 31 - 1] + [g % Gs for g in range(Gd - 6)], np.int32)
    dst.gather(src, idx)
    _l.check(E._lib, E._lib.elfb200_gather_games_dev(dst._ctx, src._ctx, idx.ctypes.data))
    dst.features(), dst.features_df(), dst.legal_mask(), dst.info()
    assert (dst.getHashCode()[2:4] == src.getHashCode()[[0, Gs - 1]]).all()
    src.close(), dst.close()
print("ASAN GATHER CLEAN")
"""


def test_gather_clean_under_address_sanitizer(emu):
    """the copy with negative and out-of-range indices on the emulator build under AddressSanitizer (every
    device buffer is a heap allocation there, so any read or write outside a batch is reported)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        asan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        pytest.skip(f"no gcc: {e}")
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("libasan is not installed")
    env = dict(os.environ, LD_PRELOAD=os.path.realpath(asan), ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0")
    r = subprocess.run([sys.executable, "-c", _ASAN_CHILD, root], env=env, capture_output=True, text=True, timeout=850)
    assert r.returncode == 0 and "ASAN GATHER CLEAN" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]
