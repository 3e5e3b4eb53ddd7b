"""Pass-alive chains and areas on the H100: k_pass_alive on full batches of eye-avoiding random-policy positions
against tests/benson_ref.py point for point, the host and device forms against each other, board.pass_alive(out=...)
after GoEnv.step in a captured CUDA graph against the same loop run eagerly, the owner-passes property on a full
batch, and final_status(pass_alive=True) against the restated rule and the reference's getTrompTaylorScore.  The
same checks run on the SIMT emulator in tests/test_pass_alive.py."""
import multiprocessing as mp
import os

import numpy as np
import pytest

from tests import oracles
from tests import test_pass_alive as TP

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def _corpus(n, G, max_plies, seed):
    """(move lists, stones, expected alive, expected area) of G games, played and restated in worker processes
    (before CUDA is touched)"""
    chunk = 64
    jobs = [(n, seed * 100003 + i, min(chunk, G - i), max_plies) for i in range(0, G, chunk)]
    with mp.get_context("fork").Pool(min(len(jobs), os.cpu_count() or 1)) as pool:
        parts = pool.map(TP.corpus_chunk, jobs)
    return ([m for p in parts for m in p[0]],) + tuple(np.concatenate([p[j] for p in parts]) for j in (1, 2, 3))


_cache = {}


def corpus(n, kind):
    key = (n, kind)
    if key not in _cache:
        G = 16384 if n == 9 else 4096
        _cache[key] = _corpus(n, G, None if kind == "end" else 150, seed=n + (kind == "mid"))
    return _cache[key]


@pytest.fixture(scope="module", autouse=True)
def _restated_first():
    """every corpus is played and restated before this module touches CUDA"""
    for key in ((19, "end"), (19, "mid"), (9, "end")):
        corpus(*key)


@pytest.mark.parametrize("n,kind", [(19, "end"), (19, "mid"), (9, "end")])
def test_full_batches_match_restatement(n, kind):
    import torch

    import elf_b200

    lists, stones, ea, er = corpus(n, kind)
    gb = elf_b200.GoBatch(len(lists), board_size=n)
    gb.replay(lists)
    h0, i0, l0 = gb.getHashCode(), gb.info(), gb.legal_mask()
    np.testing.assert_array_equal(gb.stones(), stones)
    alive, area = gb.pass_alive()
    bad = np.argwhere((alive != ea) | (area != er))
    assert len(bad) == 0, f"{len(bad)} points differ, first (game, action) {bad[:5].tolist()}"
    TP.check_invariants(stones, alive, area)
    if kind == "end":
        assert alive.sum() > 0 and (area > 0).sum() > 0
    np.testing.assert_array_equal(gb.getHashCode(), h0)
    np.testing.assert_array_equal(gb.info(), i0)
    np.testing.assert_array_equal(gb.legal_mask(), l0)
    # the device form gives the same values, each output alone too
    at = torch.full(alive.shape, 9, dtype=torch.uint8, device="cuda")
    rt = torch.full(area.shape, 9, dtype=torch.uint8, device="cuda")
    assert gb.pass_alive(out=(at, rt)) == (at, rt)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(at.cpu().numpy(), alive)
    np.testing.assert_array_equal(rt.cpu().numpy(), area)
    rt.fill_(9)
    gb.pass_alive(out=(None, rt))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(rt.cpu().numpy(), area)
    # final_status(pass_alive=True): the restated rule with and without counts; the reference scorer on a sample
    refs = None
    if oracles.have_ref(n):
        refs = []
        for mv in lists[:256]:
            r = oracles.Ref(n)
            for a in mv:
                r.forward(a)
            refs.append(r)
    counts = gb.ownership(8, seed=5)
    for c, k in ((None, None), (counts, 8)):
        base = gb.final_status(c, k, 0.5)
        dead, terr, score = gb.final_status(c, k, 0.5, pass_alive=True)
        np.testing.assert_array_equal(dead, TP.expected_dead(stones, alive, area, base[0] if c is not None else None))
        if refs is not None:
            from tests.test_ownership import ref_tt_territory

            for g, r in enumerate(refs):
                et, es = ref_tt_territory(r, dead[g])
                np.testing.assert_array_equal(terr[g], et, err_msg=f"territory of game {g}")
                assert score[g] == es
    gb.close()


def test_owner_passes_on_a_full_batch():
    import elf_b200

    n = 19
    lists, _, ea, _ = corpus(n, "end")
    keep = [g for g in range(len(lists)) if ea[g].any()]
    lists = [list(lists[g]) for g in keep]
    for mv in lists:  # drop the closing passes, so that the game goes on from the same stones
        while mv and mv[-1] == n * n:
            mv.pop()
    gb = elf_b200.GoBatch(len(lists), board_size=n)
    gb.replay(lists)
    alive, _ = gb.pass_alive()
    np.testing.assert_array_equal(alive, ea[keep])
    # the opponent moves until it has no legal move left or the game reaches the ply cap
    assert TP.owner_passes_property(gb, alive, np.random.default_rng(11), plies=200) >= len(lists)
    gb.close()


def test_pass_alive_after_env_step_in_a_cuda_graph():
    """32 plies of policy -> GoEnv.step -> board.pass_alive(out=...) captured once and replayed twice, against the
    same loop run eagerly from the same start on a second batch: the alive and area tensors of every ply are
    equal"""
    import torch

    from elf_b200.env import GoEnv, random_legal_actions

    n, G, plies = 9, 1024, 32
    envs = [GoEnv.create(G, board_size=n) for _ in range(2)]
    counters = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(2)]
    outs = [(torch.zeros((plies, G, n * n), dtype=torch.uint8, device="cuda"),
             torch.zeros((plies, G, n * n), dtype=torch.uint8, device="cuda")) for _ in range(2)]
    random_legal_actions(torch.ones((G, n * n + 1), dtype=torch.bool, device="cuda"),
                         torch.zeros(1, dtype=torch.int64, device="cuda"))  # warm-up outside the capture

    def loop(i, obs):
        for t in range(plies):
            obs = envs[i].step(random_legal_actions(obs["legal"], counters[i], seed=3))
            envs[i].board.pass_alive(out=(outs[i][0][t], outs[i][1][t]))
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
        alive, area = envs[0].board.pass_alive()
        np.testing.assert_array_equal(outs[0][0][-1].cpu().numpy(), alive)
        np.testing.assert_array_equal(outs[0][1][-1].cpu().numpy(), area)
    for e in envs:
        e.close()
