"""The device-resident environment (elfb200_env_step / elfb200_reset_dev / elfb200_observe_dev, k_env_step,
elf_b200.env.GoEnv) against the compiled reference, with one reference GoState per game.

CPU: the kernels run on the SIMT emulator build of the kernel sources (tests/simt_emu), under every lane
order; the GoEnv tensors are CPU tensors there.  tests/test_zz_gpu_env.py runs the same checks on an H100."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from tests import oracles
from tests.test_handicap import need_ref, ref_place_handicap

pytestmark = pytest.mark.timeout(900)

KOMI = 7.5
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def to_np(t):
    return t.cpu().numpy()


def ref_info(r):
    i = r.info()
    i[8] = 0  # ko_age is not part of the device state
    return i


def pick_actions(rng, refs, n, p_pass=0.08):
    """per game: mostly a uniform legal non-eye move, sometimes a pass (often enough that games also end
    by two passes), an arbitrary point (often occupied or illegal), or -1 (game left as it is)"""
    acts = np.empty(len(refs), np.int32)
    for g, r in enumerate(refs):
        u = rng.random()
        cand = np.flatnonzero(r.legal() & (1 - r.true_eyes(int(r.info()[1]))))
        if u < p_pass or len(cand) == 0:
            acts[g] = n * n
        elif u < p_pass + 0.03:
            acts[g] = int(rng.integers(0, n * n))
        elif u < p_pass + 0.05:
            acts[g] = -1
        else:
            acts[g] = int(rng.choice(cand))
    return acts


def assert_obs(env, obs, refs, label):
    """legal mask, info words and hash of every game equal its reference state"""
    n = env.board_size
    legal, info, h = to_np(obs["legal"]), to_np(obs["info"]), env.board.getHashCode()
    for g, r in enumerate(refs):
        np.testing.assert_array_equal(legal[g, :-1], r.legal().astype(bool), err_msg=f"legal g={g} {label}")
        assert legal[g, n * n], f"pass g={g} {label}"
        np.testing.assert_array_equal(info[g], ref_info(r), err_msg=f"info g={g} {label}")
        assert int(h[g]) == r.hash(), f"hash g={g} {label}"


def end_reason(r):
    """why a terminated reference game ended"""
    i = r.info()
    return "superko" if i[11] else "two_pass" if i[10] else "ply_cap"


def step_and_check(env, refs, acts, d4, label):
    """one env step against the reference: ok, done, value (bit for bit, taken before the reference is
    replaced), then a fresh reference where done; returns (obs, done, the end reasons seen)"""
    obs = env.step(torch.from_numpy(acts).to(env.device), None if d4 is None else torch.from_numpy(d4).to(env.device))
    ok, done, value = to_np(obs["ok"]), to_np(obs["done"]).astype(bool), to_np(obs["value"])
    reasons = []
    for g, (r, a) in enumerate(zip(refs, acts)):
        want_ok = r.forward(int(a)) if a >= 0 else False
        assert bool(ok[g]) == want_ok, f"ok g={g} a={a} {label}"
        assert done[g] == r.terminated(), f"done g={g} {label}"
        if done[g]:
            want = np.float32(r.evaluate(KOMI))
            assert value[g].tobytes() == want.tobytes(), f"value g={g} {value[g]} != {want} {label}"
            reasons.append(end_reason(r))
            refs[g] = oracles.Ref(env.board_size)
        else:
            assert value[g] == 0.0
    return obs, done, reasons


def run_env_parity(make_env, n, G, seed, rounds=2):
    """G games (9x9: three per warp) under a random policy with illegal, occupied, untouched and pass actions,
    until every game has finished at least `rounds` times.  After every step ok / done / value / legal / info
    / hash equal the reference; the AGZ planes under random D4 codes every 10 plies and on the two plies
    after a restart (the history planes are zero at ply 1), and the DarkForest planes of restarted games
    (the `placed` array was cleared)."""
    rng = np.random.default_rng(seed)
    env = make_env(G, n, features="f32")
    refs = [oracles.Ref(n) for _ in range(G)]
    obs = env.reset()
    assert_obs(env, obs, refs, "reset")
    finished = np.zeros(G, int)
    since = np.full(G, 99)  # plies since the last restart
    reasons, mixed_warp = set(), False
    t = 0
    while finished.min() < rounds:
        acts = pick_actions(rng, refs, n)
        d4 = rng.integers(0, 8, G).astype(np.int32)
        obs, done, rs = step_and_check(env, refs, acts, d4, f"ply {t}")
        reasons |= set(rs)
        finished += done
        since = np.where(done, 0, since + 1)
        assert_obs(env, obs, refs, f"ply {t}")
        if n == 9:
            w = done[: G // 3 * 3].reshape(-1, 3)
            mixed_warp |= bool((w.any(1) & ~w.all(1)).any())
        fresh = since <= 1
        if t % 10 == 0 or fresh.any():
            planes = to_np(obs["planes"])
            for g in range(G) if t % 10 == 0 else np.flatnonzero(fresh):
                np.testing.assert_array_equal(planes[g], refs[g].features(int(d4[g])), err_msg=f"AGZ g={g} ply {t}")
            for g in np.flatnonzero(done):
                assert (planes[g, :16] == 0).all()
        if (since == 2).any():
            df = env.board.features_df(d4)
            for g in np.flatnonzero(since == 2):
                np.testing.assert_array_equal(df[g], refs[g].features_df(int(d4[g])), err_msg=f"DF g={g} ply {t}")
        t += 1
        assert t < 20 * n * n
    assert "two_pass" in reasons
    if n == 9:
        assert mixed_warp  # a game ended on a step where another game of its warp did not
    env.close()
    return reasons


def run_end_reasons(make_env):
    """the three ways a game ends, each scored and restarted: two passes, positional superko (the golden
    capture cycle), the 2N^2 ply cap (a game that fills its own eyes), and a game that had already ended
    through the host step API before the env step"""
    n = 9
    P = n * n
    opening = json.load(open(os.path.join(GOLDEN, "mcts_superko_opening_9.json")))["openings"][0]
    env = make_env(4, n)
    refs = [oracles.Ref(n) for _ in range(4)]
    env.reset()
    # game 0: two passes at once; game 1: the superko opening and the recapture 4, 3 that closes the cycle;
    # game 2: two moves and two passes, then the same two moves again (a superko record left from the first
    # game would hold the position after the first move); game 3: ended by two host-side passes, then an env
    # step with a move
    seq1 = opening + [4, 3]
    seq2 = [40, 41, P, P, 40, 41]
    env.board.forward(np.array([-1, -1, -1, P], np.int32))
    env.board.forward(np.array([-1, -1, -1, P], np.int32))
    refs[3].forward(P)
    refs[3].forward(P)
    assert env.board.terminated()[3]
    seen = {}
    for t in range(len(seq1)):
        acts = np.array([P if t < 2 else -1, seq1[t], seq2[t] if t < len(seq2) else -1, 20 if t == 0 else -1],
                        np.int32)
        _, done, rs = step_and_check(env, refs, acts, None, f"ply {t}")
        for g, why in zip(np.flatnonzero(done), rs):
            assert g not in seen
            seen[g] = (t, why)
    assert seen == {0: (1, "two_pass"), 1: (len(seq1) - 1, "superko"), 2: (3, "two_pass"), 3: (0, "two_pass")}
    assert to_np(env.info)[2, 0] == 3 and not to_np(env.info)[2, 11]
    # the superko: +1 for black to move after white's recapture; the game restarted
    assert to_np(env.value)[1] == 1.0 and to_np(env.info)[1, 0] == 1
    env.close()
    # the ply cap: uniform legal moves, pass only when nothing else is legal; this seed's game 0 fills its
    # eyes and reaches 2N^2 = 162 plies
    env = make_env(3, n)
    refs = [oracles.Ref(n) for _ in range(3)]
    obs = env.reset()
    counter = torch.zeros(1, dtype=torch.int64, device=env.device)
    from elf_b200.env import random_legal_actions

    caps = []
    for t in range(2 * P):
        acts = to_np(random_legal_actions(obs["legal"], counter, seed=CAP_SEED))
        pre = [r.info().copy() for r in refs]
        obs, done, rs = step_and_check(env, refs, acts, None, f"cap ply {t}")
        caps += [g for g, r in zip(np.flatnonzero(done), rs) if r == "ply_cap"]
        if 0 in caps:
            assert t == 2 * P - 2 and pre[0][0] == 2 * P - 1
            break
    assert 0 in caps
    env.close()


CAP_SEED = 3


def run_mask_reset_and_observe(make_env):
    """elfb200_reset_dev restarts only the masked games; elfb200_observe_dev after elfb200_place_handicap
    gives the handicap positions' legal masks and info words"""
    n, G = 9, 5
    rng = np.random.default_rng(5)
    env = make_env(G, n)
    refs = [oracles.Ref(n) for _ in range(G)]
    env.reset()
    for t in range(12):
        step_and_check(env, refs, pick_actions(rng, refs, n, p_pass=0.0), None, f"ply {t}")
    mask = np.array([1, 0, 0, 1, 0], bool)
    obs = env.reset(torch.from_numpy(mask).to(env.device))
    refs = [oracles.Ref(n) if m else r for m, r in zip(mask, refs)]
    assert_obs(env, obs, refs, "masked reset")
    assert not to_np(obs["done"]).any() and not to_np(obs["ok"]).any()
    obs = env.reset(torch.from_numpy(np.array([0, 1, 0, 0, 0], np.uint8)).to(env.device))
    refs[1] = oracles.Ref(n)
    assert_obs(env, obs, refs, "uint8 mask")
    # handicap positions: the first observation comes from elfb200_observe_dev
    env.reset()
    refs = [oracles.Ref(n) for _ in range(G)]
    lists = [[20, 60], [], [40], [10, 10, 70], [0, 1, 2, 3]]
    ok = env.board.place_handicap(lists)
    for g, (r, s) in enumerate(zip(refs, lists)):
        assert ok[g].tolist() == [ref_place_handicap(r, a) for a in s]
    assert_obs(env, env.observe(), refs, "handicap")
    for t in range(6):
        step_and_check(env, refs, pick_actions(rng, refs, n), None, f"handicap ply {t}")
        assert_obs(env, env.obs, refs, f"handicap ply {t}")
    env.close()


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

    return make


@pytest.mark.parametrize("n,G", [(9, 50), (19, 8)])
def test_env_matches_reference_every_ply(make_env, lane_order, n, G):
    need_ref(n)
    run_env_parity(make_env, n, G, seed=11 * n)


def test_env_end_reasons(make_env, lane_order):
    need_ref(9)
    run_end_reasons(make_env)


def test_env_mask_reset_and_observe(make_env, lane_order):
    need_ref(9)
    run_mask_reset_and_observe(make_env)


ERR_ARG = -1  # ELFB200_ERR_ARG (include/elfb200.h)


def test_env_step_arguments(emu):
    L = emu.emu_lib()
    gb = emu.emu_batch(4, 9)
    acts = np.array([40, 81, -1, 3], np.int32)
    out8 = np.zeros(4 * 82, np.uint8)
    assert L.elfb200_env_step(None, acts.ctypes.data, 7.5, None, None, None, None, None) == ERR_ARG
    assert L.elfb200_env_step(gb._ctx, None, 7.5, out8.ctypes.data, None, None, None, None) == ERR_ARG
    assert L.elfb200_reset_dev(None, None) == ERR_ARG and L.elfb200_observe_dev(None, None, None) == ERR_ARG
    assert not out8.any()
    # every output NULL: the games still move
    assert L.elfb200_env_step(gb._ctx, acts.ctypes.data, 7.5, None, None, None, None, None) == 0
    assert gb.info()[:, 0].tolist() == [2, 2, 1, 2]
    assert L.elfb200_observe_dev(gb._ctx, None, None) == 0 and L.elfb200_reset_dev(gb._ctx, None) == 0
    assert (gb.getHashCode() == 0).all()
    gb.close()


def test_goenv_host_logic(emu):
    from elf_b200.env import GoEnv

    n, G = 9, 4
    env = GoEnv(emu.emu_batch(G, n), device="cpu")
    obs = env.reset()
    assert set(obs) == {"ok", "done", "value", "legal", "info", "planes"} and obs["planes"] is None
    for k, dt, shape in (("ok", torch.uint8, (G,)), ("done", torch.uint8, (G,)), ("value", torch.float32, (G,)),
                         ("legal", torch.bool, (G, n * n + 1)), ("info", torch.int32, (G, 12))):
        assert obs[k].dtype == dt and tuple(obs[k].shape) == shape, k
    assert obs["legal"].data_ptr() == env._legal.data_ptr() and obs["legal"].all()
    ptrs = {k: v.data_ptr() for k, v in obs.items() if v is not None}
    obs2 = env.step(torch.tensor([40, 81, -1, 40], dtype=torch.int32))
    assert obs2 is obs and {k: v.data_ptr() for k, v in obs2.items() if v is not None} == ptrs
    assert obs["ok"].tolist() == [1, 1, 0, 1] and not obs["legal"][0, 40] and obs["legal"][2, 40]
    assert obs["info"][:, 0].tolist() == [2, 2, 1, 2]
    obs = env.reset(torch.tensor([True, False, False, False]))
    assert obs["info"][:, 0].tolist() == [1, 2, 1, 2] and not obs["ok"].any()
    for bad in (torch.tensor([1, 2, 3, 4]), torch.zeros(3, dtype=torch.int32), torch.zeros((4, 1), dtype=torch.int32)):
        with pytest.raises(ValueError):
            env.step(bad)
    with pytest.raises(ValueError):
        env.reset(torch.zeros(4, dtype=torch.int32))
    with pytest.raises(ValueError):
        GoEnv(env.board, features="f64", device="cpu")
    for fmt, dt, shape in (("f32", torch.float32, (G, 18, n, n)), ("f16", torch.float16, (G, n, n, 32)),
                           ("bf16", torch.bfloat16, (G, n, n, 32))):
        e = GoEnv(env.board, features=fmt, cpad=32, device="cpu")
        p = e.reset()["planes"]
        assert p.dtype == dt and tuple(p.shape) == shape
        e.step(torch.tensor([n * n] * G, dtype=torch.int32))
        want = env.board.features()
        got = p.float() if fmt == "f32" else p[..., :18].float().permute(0, 3, 1, 2)
        np.testing.assert_array_equal(got.numpy(), want)
    env.board.close()
