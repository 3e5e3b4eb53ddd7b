"""The device-resident environment on the H100: the reference parity of tests/test_env.py through the same
run functions, full-size batches played past 2N^2 plies and replayed game by game through the reference,
and a CUDA graph of policy -> GoEnv.step against the same loop run eagerly."""
import numpy as np
import pytest
import torch

from tests import oracles
from tests.test_env import KOMI, need_ref, run_end_reasons, run_env_parity, run_mask_reset_and_observe

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def make_env(G, n, **kw):
    from elf_b200.env import GoEnv

    return GoEnv.create(G, board_size=n, **kw)


@pytest.mark.parametrize("n,G", [(9, 50), (19, 8)])
def test_env_matches_reference_every_ply(n, G):
    need_ref(n)
    run_env_parity(make_env, n, G, seed=11 * n)


def test_env_end_reasons():
    need_ref(9)
    run_end_reasons(make_env)


def test_env_mask_reset_and_observe():
    need_ref(9)
    run_mask_reset_and_observe(make_env)


@pytest.mark.parametrize("n,G", [(19, 4096), (9, 12288)])
def test_env_at_scale_matches_reference(n, G):
    """2N^2 + 50 plies of the seeded device policy, so every slot finishes a game and restarts; the
    actions, ok flags, done flags and values are logged on the device, then every slot's action stream is
    replayed through reference states: accept flags, the games finished, each value and the final hashes
    agree game by game"""
    from elf_b200.env import random_legal_actions

    need_ref(n)
    P = n * n
    T = 2 * P + 50
    env = make_env(G, n)
    obs = env.reset()
    counter = torch.zeros(1, dtype=torch.int64, device=env.device)
    log_a = torch.empty((T, G), dtype=torch.int32, device=env.device)
    log_ok, log_done = torch.empty_like(log_a, dtype=torch.uint8), torch.empty_like(log_a, dtype=torch.uint8)
    log_v = torch.empty((T, G), dtype=torch.float32, device=env.device)
    for t in range(T):
        a = random_legal_actions(obs["legal"], counter, seed=17)
        log_a[t] = a
        obs = env.step(a)
        log_ok[t], log_done[t], log_v[t] = obs["ok"], obs["done"], obs["value"]
    acts, ok, done, val = (x.cpu().numpy() for x in (log_a, log_ok, log_done, log_v))
    h = env.board.getHashCode()
    assert done.any(0).all()  # every slot finished at least one game
    games = 0
    for g in range(G):
        r = oracles.Ref(n)
        for t in range(T):
            assert r.forward(int(acts[t, g])) == bool(ok[t, g]), (g, t)
            assert r.terminated() == bool(done[t, g]), (g, t)
            if done[t, g]:
                assert val[t, g].tobytes() == np.float32(r.evaluate(KOMI)).tobytes(), (g, t)
                games += 1
                r = oracles.Ref(n)
        assert int(h[g]) == r.hash(), g
    assert games == int(done.sum()) and ok.all()
    env.close()


def test_env_cuda_graph_equals_eager():
    """32 plies of policy -> GoEnv.step (fp16 planes) captured once, replayed twice; the same loop run
    eagerly from the same start on a second batch: hashes, done, value, legal, info and planes are bitwise
    equal after 32 and after 64 plies"""
    from elf_b200.env import random_legal_actions

    n, G = 19, 4096
    graph_env, eager_env = make_env(G, n, features="f16"), make_env(G, n, features="f16")
    c_graph = torch.zeros(1, dtype=torch.int64, device="cuda")
    c_eager = torch.zeros(1, dtype=torch.int64, device="cuda")
    # warm the policy's kernels up outside the capture
    random_legal_actions(torch.ones((G, n * n + 1), dtype=torch.bool, device="cuda"),
                         torch.zeros(1, dtype=torch.int64, device="cuda"))
    obs = graph_env.reset()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(32):
            obs = graph_env.step(random_legal_actions(obs["legal"], c_graph, seed=5))
    eobs = eager_env.reset()
    for rep in range(2):
        graph.replay()
        for _ in range(32):
            eobs = eager_env.step(random_legal_actions(eobs["legal"], c_eager, seed=5))
        torch.cuda.synchronize()
        assert (graph_env.board.getHashCode() == eager_env.board.getHashCode()).all(), rep
        for k in ("ok", "done", "value", "legal", "info", "planes"):
            assert torch.equal(obs[k], eobs[k]), (k, rep)
        assert int(c_graph) == int(c_eager) == 32 * (rep + 1)
    assert (graph_env.board.getPly() > 1).any()
    graph_env.close()
    eager_env.close()
