"""Ladders and self-ataris on the H100: k_tactics on every position of the ladder suite and on full batches of
random positions against the compiled reference, triple for triple, the host and device forms against each other,
and board.tactics(out=...) after GoEnv.step in a captured CUDA graph against the same loop run eagerly.  The same
checks run on the SIMT emulator in tests/test_tactics.py."""
import multiprocessing as mp
import os

import numpy as np
import pytest

from tests import tactics_ref as T
from tests.test_handicap import need_ref

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def _reference(n, lists):
    """reference (ladder, self_atari, calls) of every move list, in worker processes (before CUDA is touched)"""
    chunk = 128
    jobs = [(n, lists[i:i + chunk], False) for i in range(0, len(lists), chunk)]
    with mp.get_context("fork").Pool(min(len(jobs), os.cpu_count() or 1)) as pool:
        parts = pool.map(T.ref_chunk, jobs)
    return tuple(np.concatenate([p[j] for p in parts]) for j in range(3))


def _random_lists(n, G, plies, seed):
    """G games of `plies` uniform legal moves (fewer if one ends), played on the reference"""
    rng = np.random.default_rng(seed)
    return [T.random_game(n, rng, plies) for _ in range(G)]


def _check(n, lists):
    import elf_b200

    need_ref(n)
    exp = _reference(n, lists)
    gb = elf_b200.GoBatch(len(lists), board_size=n)
    gb.replay(lists)
    h0, i0, l0 = gb.getHashCode(), gb.info(), gb.legal_mask()
    got = gb.tactics(trace=True)
    for name, a, b in zip(("ladder", "self_atari", "calls"), got, exp):
        bad = np.argwhere(a != b)
        assert len(bad) == 0, f"{name}: {len(bad)} triples differ, first {bad[:5].tolist()}"
    np.testing.assert_array_equal(gb.getHashCode(), h0)
    np.testing.assert_array_equal(gb.info(), i0)
    np.testing.assert_array_equal(gb.legal_mask(), l0)
    assert (got[0] >= 0).all()
    return gb, got


def test_ladder_suite_in_one_batch_matches_reference():
    import torch

    lists = T.ladder_suite_lists()
    assert len(lists) == 12522
    gb, (lad, sa, calls) = _check(19, lists)
    assert (lad > 0).sum() >= 1500 and (calls > 0).sum() >= 3500
    # the device form gives the same values
    lt = torch.full(lad.shape, -7, dtype=torch.int16, device="cuda")
    st = torch.full(sa.shape, -7, dtype=torch.int16, device="cuda")
    assert gb.tactics(out=(lt, st)) == (lt, st)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(lt.cpu().numpy(), lad)
    np.testing.assert_array_equal(st.cpu().numpy(), sa)
    lt.fill_(-7)
    gb.tactics(out=(lt, None))  # one output alone
    torch.cuda.synchronize()
    np.testing.assert_array_equal(lt.cpu().numpy(), lad)
    gb.close()


@pytest.mark.parametrize("n,G,plies", [(19, 4096, 150), (9, 12288, 40)])
def test_random_positions_match_reference(n, G, plies):
    _check(n, _random_lists(n, G, plies, seed=7 * n))[0].close()


def test_tactics_after_env_step_in_a_cuda_graph():
    """32 plies of policy -> GoEnv.step -> board.tactics(out=...) captured once and replayed twice, against the
    same loop run eagerly from the same start on a second batch: the ladder and self-atari tensors of every ply
    are equal"""
    import torch

    from elf_b200.env import GoEnv, random_legal_actions

    n, G, plies = 19, 1024, 32
    envs = [GoEnv.create(G, board_size=n) for _ in range(2)]
    counters = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(2)]
    outs = [(torch.zeros((plies, G, 2, n * n), dtype=torch.int16, device="cuda"),
             torch.zeros((plies, G, 2, n * n), dtype=torch.int16, device="cuda")) for _ in range(2)]
    random_legal_actions(torch.ones((G, n * n + 1), dtype=torch.bool, device="cuda"),
                         torch.zeros(1, dtype=torch.int64, device="cuda"))  # warm-up outside the capture

    def loop(i, obs):
        for t in range(plies):
            obs = envs[i].step(random_legal_actions(obs["legal"], counters[i], seed=3))
            envs[i].board.tactics(out=(outs[i][0][t], outs[i][1][t]))
        return obs

    obs = envs[0].reset()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loop(0, obs)
    eobs = envs[1].reset()
    for rep in range(2):
        graph.replay()
        eobs = loop(1, eobs)
        torch.cuda.synchronize()
        assert (envs[0].board.getHashCode() == envs[1].board.getHashCode()).all(), rep
        for k in range(2):
            assert torch.equal(outs[0][k], outs[1][k]), (k, rep)
        # the last ply's tensors are those of the host form on the position it left
        lad, sa = envs[0].board.tactics()
        np.testing.assert_array_equal(outs[0][0][-1].cpu().numpy(), lad)
        np.testing.assert_array_equal(outs[0][1][-1].cpu().numpy(), sa)
    assert (outs[0][1] > 0).any()
    for e in envs:
        e.close()
