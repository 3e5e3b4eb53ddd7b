"""Monte-Carlo ownership and dead stones on the H100: k_ownership at full batch size against the compiled reference
playout by playout, the device form captured in a CUDA graph, and GTP final_status_list on the real board.  The
same checks run on the SIMT emulator in tests/test_ownership.py."""
import multiprocessing as mp
import os

import numpy as np
import pytest

from tests import oracles
from tests.test_handicap import BatchStubSearch, need_ref
from tests.test_ownership import ref_playout_from, run_gtp_final_status

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def _move_lists(n, G, plies, rng):
    """G lists of `plies` random actions (a few passes); replay skips the ones the board refuses, as the reference's
    switchBeforeMove does"""
    P = n * n
    acts = rng.integers(0, P, (G, plies))
    acts[rng.random((G, plies)) < 0.01] = P
    return [list(map(int, row)) for row in acts]


def _ref_chunk(args):
    """reference side of games g0.. : (plies [g][K], final hash [g][K], counts [g][2][P])"""
    n, lists, g0, K, seed = args
    P = n * n
    plies = np.zeros((len(lists), K), np.int32)
    hashes = np.zeros((len(lists), K), np.uint64)
    counts = np.zeros((len(lists), 2, P), np.int32)
    for i, lst in enumerate(lists):
        r = oracles.Ref(n)
        for a in lst:
            r.forward(a)
        for k in range(K):
            t, h, terr, _ = ref_playout_from(r, seed, (g0 + i) * K + k, 2 * P)
            plies[i, k], hashes[i, k] = t, h
            counts[i, 0] += terr == 1
            counts[i, 1] += terr == 2
    return plies, hashes, counts


def _reference(n, lists, K, seed):
    chunk = 64
    jobs = [(n, lists[i:i + chunk], i, K, seed) for i in range(0, len(lists), chunk)]
    with mp.get_context("fork").Pool(min(len(jobs), os.cpu_count() or 1)) as pool:
        parts = pool.map(_ref_chunk, jobs)
    return tuple(np.concatenate([p[j] for p in parts]) for j in range(3))


@pytest.mark.parametrize("n,G,plies,K", [(19, 4096, 150, 4), (9, 12288, 40, 2)])
def test_ownership_at_scale_matches_reference(n, G, plies, K):
    import elf_b200

    need_ref(n)
    rng = np.random.default_rng(5 * n)
    lists = _move_lists(n, G, plies, rng)
    exp_plies, exp_hash, exp_counts = _reference(n, lists, K, seed=21)  # before CUDA is touched (fork)
    gb = elf_b200.GoBatch(G, board_size=n)
    gb.replay(lists)
    counts, fh, pl = gb.ownership(K, seed=21, trace=True)
    np.testing.assert_array_equal(pl, exp_plies)
    np.testing.assert_array_equal(fh, exp_hash)
    np.testing.assert_array_equal(counts, exp_counts)
    np.testing.assert_array_equal(gb.ownership(K, seed=21), counts)  # the same counts on a second run
    gb.close()


def test_ownership_captured_in_a_cuda_graph():
    import torch

    import elf_b200

    n, G, K = 19, 256, 8
    gb = elf_b200.GoBatch(G, board_size=n)
    gb.replay(_move_lists(n, G, 120, np.random.default_rng(3)))
    want = gb.ownership(K, seed=9)  # also sets up the scratch
    out = torch.full((G, 2, n * n), -1, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        gb.ownership(K, seed=9, out=out)  # warm-up of the device form outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), want)
    out.fill_(-1)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gb.ownership(K, seed=9, out=out)
    graph.replay()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), want)
    gb.close()


def test_gtp_final_status_list_on_the_real_board():
    """the constructed 9x9 endgame entered with GTP play commands and two passes: final_status_list answers as
    the emulator does for the same position and seed"""
    import torch

    import elf_b200
    from elf_b200 import console, online

    need_ref(9)
    gb = elf_b200.GoBatch(1, board_size=9)
    g = online.OnlineGame(gb, BatchStubSearch(gb))
    c = console.GtpConsole(g, lambda batch: {"pi": torch.ones(batch["s"].shape[0], 82), "V": torch.zeros(1)})
    c.final_status_playouts = 256
    got = run_gtp_final_status(g, c)
    try:
        from tests import emu as E

        E.emu_lib()
    except Exception as e:
        pytest.skip(f"SIMT emulator build unavailable: {e}")
    eb = E.emu_batch(1, 9)
    eg = online.OnlineGame(eb, BatchStubSearch(eb))
    ec = console.GtpConsole(eg, None)
    ec.final_status_playouts = c.final_status_playouts
    assert run_gtp_final_status(eg, ec) == got
