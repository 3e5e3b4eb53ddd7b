"""Handicap stones on the H100: elfb200_place_handicap (k_place) against the compiled reference, whole
games from handicap positions at full batch size, the search from handicap roots, and one online
handicap game with a 20x256 network.  The same board and search checks run on the SIMT emulator in
tests/test_handicap.py."""
import numpy as np
import pytest

from tests import oracles
from tests.test_handicap import SEARCH_OPTS, need_ref, ref_place_handicap, run_board_parity, run_search_from_handicap

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _gobatch(G, n):
    import elf_b200

    return elf_b200.GoBatch(G, board_size=n)


@pytest.mark.parametrize("n", [9, 19])
def test_place_handicap_matches_reference_every_ply(n):
    need_ref(n)
    run_board_parity(_gobatch, n, seed=40 + n, max_plies=2 * n * n + 10)


@pytest.mark.parametrize("n,G", [(19, 4096), (9, 12288)])
def test_handicap_games_to_the_end_at_scale(n, G):
    """G games with random handicaps (none, the GTP fixed placements, random free lists) are played to
    the end through the step API with a seeded random policy over the device's legal non-eye moves; the
    reference plays the same moves.  Per ply the accept flags, at the end hash, captures, ply and score
    agree game by game."""
    from elf_b200.console import fixed_handicap_vertices
    from elf_b200.online import vertex2action

    need_ref(n)
    P = n * n
    rng = np.random.default_rng(7 * n)
    gb = _gobatch(G, n)
    refs = [oracles.Ref(n) for _ in range(G)]
    lists = []
    for g in range(G):
        k = int(rng.integers(0, 10))
        if k >= 2 and g % 2:
            lists.append([vertex2action(v, n) for v in fixed_handicap_vertices(k, n)])
        else:
            lists.append([int(a) for a in rng.choice(P, k, replace=False)])
    ok = gb.place_handicap(lists)
    for g, (r, s) in enumerate(zip(refs, lists)):
        assert ok[g].tolist() == [ref_place_handicap(r, a) for a in s], g
    assert sum(len(s) for s in lists) > 4 * G
    plies = 0
    while not gb.terminated().all():
        cand = gb.legal_mask()[:, :P].astype(bool) & ~gb.true_eyes(0).astype(bool)
        keys = np.where(cand, rng.random((G, P)), -1.0)
        acts = np.where(cand.any(1), keys.argmax(1), P).astype(np.int32)
        acts[gb.terminated()] = -1
        got = gb.forward(acts)
        want = [r.forward(int(a)) if a >= 0 else False for r, a in zip(refs, acts)]
        np.testing.assert_array_equal(got, want, err_msg=f"ply {plies}")
        plies += 1
        assert plies <= 2 * P + 1
    h, info, sc = gb.getHashCode(), gb.info(), gb.tt_score()
    for g, r in enumerate(refs):
        ri = r.info()
        assert (int(h[g]), info[g, 0], info[g, 2], info[g, 3], sc[g]) == (r.hash(), ri[0], ri[2], ri[3], r.tt_score()), g
    assert info[:, 2:4].sum() > 0
    gb.close()


@pytest.mark.parametrize("n,stones", [(19, (2, 4, 9)), (9, (4,))])
def test_search_from_handicap_matches_reference(n, stones):
    import elf_b200

    need_ref(n)
    run_search_from_handicap(_gobatch, elf_b200.MctsBatch, n, stones, SEARCH_OPTS)


def test_online_handicap_game_with_a_network():
    """fixed_handicap 9 on 19x19, then white (the engine, a random-init 20x256 network) and black (random
    legal moves) alternate: every reply is a legal vertex and the search reports no errors"""
    import torch

    from elf_b200 import console, online
    from elf_b200.model import Actor, PolicyValueNet

    n = 19
    torch.manual_seed(0)
    net = PolicyValueNet(n, num_block=20, dim=256).cuda()
    g = online.OnlineGame.create(board_size=n, num_rollouts=128, num_rollouts_per_batch=16, c_puct=1.5,
                                 virtual_loss=1, persistent_tree=1, rotation_flip=1)
    c = console.GtpConsole(g, Actor(net, batchsize=16))
    assert c.execute("fixed_handicap 9") == "= D4 Q16 D16 Q4 D10 Q10 K4 K16 K10\n\n"
    rng = np.random.default_rng(0)
    for t in range(20):
        legal = g.board.legal_mask()[0]
        r = c.execute("genmove w")
        assert r.startswith("= ") and r.endswith("\n\n"), r
        v = r[2:-2]
        assert v == "PASS" or legal[online.vertex2action(v, n)], (t, v)
        a = int(rng.choice(np.flatnonzero(g.board.legal_mask()[0][: n * n])))
        assert c.execute(f"play b {online.action2vertex(a, n)}") == "=\n\n"
        assert (g.search.errors() == 0).all()
    assert g.info()[0] == 41 and g.finished == []
