"""The search on the DarkForest planes (GameOptions::use_df_feature): k_leaf_features_df on the SIMT emulator
build of the kernel sources against the compiled reference's search with BoardFeature::extract as its
network input (oracle/ref_mcts_df_shim.cc), plus the format's other entry points and the compat surface.
tests/test_zz_gpu_df_search.py runs the same scenarios on an H100."""
import numpy as np
import pytest
import torch

from elf_b200 import lib as _l
from tests import emu
from tests.df_search import DfNet, RefWorker, callback, digest_np, have_df_ref, ko_line, random_lines, run_df_search

pytestmark = pytest.mark.timeout(1800)

OPTS = dict(num_rollouts=64, num_rollouts_per_batch=8, virtual_loss=1, persistent_tree=1, c_puct=1.5)


def need(n):
    if not have_df_ref(n):
        pytest.skip("compiled reference (oracle/_ref) not available")


def df_search(gb, **kw):
    """the emulated search with its leaf batch in the DarkForest format"""
    mc = emu.EmuSearch(gb, **kw)
    n = gb.board_size
    mc.feature_format, mc._fmt = "df", _l.FEAT_DF_F32_NCHW
    mc.feat = torch.zeros((mc.max_leaves, 25, n, n), dtype=torch.float32)
    return mc


def attach_streams(mc, seeds):
    from elf_b200.refstream import RefStream

    rs = RefStream(len(seeds), mc.gb.board_size, np.asarray(seeds, np.uint64))
    rs.init_actor(0)
    mc.attach_ref_stream(rs, 0)


def near_cap_lines(n, G, seed):
    """random games within 20 plies of the 2N^2 cap (MAX_PLY); a game that ends earlier is drawn again"""
    return random_lines(n, G, 2 * n * n - 20, seed)


SCENARIOS = {
    # name: (lines(n, G) or None, handicap(n) or None, moves)
    "fresh_after_captures": (lambda n, G: random_lines(n, G, 40 if n == 9 else 90, 11, captures=True), None, 1),
    "persistent_5_moves": (lambda n, G: random_lines(n, G, 10, 12), None, 5),
    "ko_fight": (lambda n, G: [ko_line(n)] * G, None, 3),  # with ko_callback: the fight is forced
    "handicap_ply1": (None, lambda n, G: [[a * n + b for a, b in ((2, 2), (n - 3, n - 3), (2, n - 3), (n - 3, 2))]] * G, 3),
}


@pytest.mark.parametrize("flip", [0, 1])
@pytest.mark.parametrize("scenario", sorted(SCENARIOS))
@pytest.mark.parametrize("n", [9, 19])
def test_search_equals_reference(n, scenario, flip):
    need(n)
    G = 2
    lines_f, hcap_f, moves = SCENARIOS[scenario]
    gb = emu.emu_batch(G, n)
    seeds = [20261017 + g for g in range(G)] if flip else None
    mc = df_search(gb, rotation_flip=flip, std_sort_ties=flip, **OPTS)
    if flip:
        attach_streams(mc, seeds)
    run_df_search(gb, mc, n, OPTS, moves, lines=lines_f(n, G) if lines_f else None,
                  handicap=hcap_f(n, G) if hcap_f else None, seeds=seeds,
                  net_name="ko" if scenario == "ko_fight" else "plain")


@pytest.mark.parametrize("n", [9, 19])
def test_root_near_the_ply_cap(n):
    need(n)
    G = 1
    gb = emu.emu_batch(G, n)
    mc = df_search(gb, rotation_flip=0, **OPTS)
    run_df_search(gb, mc, n, OPTS, 3, lines=near_cap_lines(n, G, 5))


@pytest.mark.parametrize("n", [9, 19])
def test_leaf_planes_bit_equal_to_reference(n):
    """every wave: our leaves matched to the reference's evaluated leaves by position hash, the 25 planes
    compared bit for bit -- a forced ko fight with a persistent tree, so paths capture a stone and play
    the same point again (the DF history planes of such a point come from the move nearest the leaf)"""
    need(n)
    G = 2
    opts = dict(OPTS, num_rollouts=128)
    gb = emu.emu_batch(G, n)
    mc = df_search(gb, rotation_flip=0, **opts)
    checked = run_df_search(gb, mc, n, opts, 4, lines=[ko_line(n)] * G, plane_check=True, net_name="ko")
    assert checked >= 4 * G * opts["num_rollouts"] // 2


@pytest.mark.parametrize("n", [9, 19])
def test_board_batch_format_equals_features_df(n):
    """elfb200_features_dev_ex(..., ELFB200_FEAT_DF_F32_NCHW) is features_df, cpad ignored"""
    G = 3
    gb = emu.emu_batch(G, n)
    for ln in zip(*random_lines(n, G, 30, 3)):
        assert gb.forward(np.array(ln, np.int32)).all()
    L = emu.emu_lib()
    d4 = np.array([0, 3, 6], np.int32)
    out = np.full((G, 25, n, n), np.nan, np.float32)
    _l.check(L, L.elfb200_features_dev_ex(gb._ctx, d4.ctypes.data, out.ctypes.data, _l.FEAT_DF_F32_NCHW, 7))
    np.testing.assert_array_equal(out.view(np.uint32), gb.features_df(d4).view(np.uint32))


def test_leaf_features_again_is_idempotent():
    n, G = 9, 2
    gb = emu.emu_batch(G, n)
    for ln in zip(*random_lines(n, G, 12, 4)):
        assert gb.forward(np.array(ln, np.int32)).all()
    mc = df_search(gb, rotation_flip=0, **OPTS)
    mc.begin_move()
    for _ in range(3):
        s = mc.select()
        k = s.shape[0]
        first = s.clone()
        again = torch.full_like(mc.feat, float("nan"))
        _l.check(mc._lib, mc._lib.elfb200_mcts_leaf_features(mc._m, again.data_ptr(), _l.FEAT_DF_F32_NCHW, 0))
        assert torch.equal(again[:k].view(torch.int32), first.view(torch.int32))
        pi, v = callback(first.numpy())
        mc.expand_backup(torch.from_numpy(pi), torch.from_numpy(v))


def test_torch_twin_equals_numpy_digest():
    n = 19
    rng = np.random.default_rng(1)
    x = rng.random((6, 25, n, n)).astype(np.float32) * 10000
    x[0] = 0
    x[1, 14] = 10000.0
    d = digest_np(x)
    t = DfNet(n, "cpu", chunk=4).digest(torch.from_numpy(x)).numpy().view(np.uint64)
    np.testing.assert_array_equal(d, t)
    y = x.copy()
    y[2, 10, 3, 4] = np.nextafter(y[2, 10, 3, 4], np.float32(1e9))
    assert digest_np(y)[2] != d[2] and (digest_np(y)[[0, 1, 3]] == d[[0, 1, 3]]).all()


def test_python_surface_rejects_and_shapes():
    from elf_b200.selfplay import SelfPlay

    with pytest.raises(ValueError, match="use_df_feature"):
        SelfPlay(None, num_games=1, board=object(), search=object(), use_df_feature=True, feature_format="f16")
    gb = emu.emu_batch(2, 9)
    from elf_b200.env import GoEnv

    env = GoEnv(gb, features="df", device="cpu")
    obs = env.reset()
    assert tuple(obs["planes"].shape) == (2, 25, 9, 9) and obs["planes"].dtype == torch.float32
    np.testing.assert_array_equal(obs["planes"].numpy(), gb.features_df())


def test_compat_contexts_report_df_planes():
    """go.GameContext(co, opt) in selfplay and online mode with use_df_feature: the flag reaches the engine,
    which reports num_planes 25 (stone planes 7 / 8) and allocates "s" as [bs,25,N,N]; without the flag the
    engine constructors see the same arguments as before"""
    from elf_b200 import compat

    got = {}

    class FakeSelfPlay:
        def __init__(self, **kw):
            got.clear()
            got.update(kw)
            self.N, self.G, self.resign_thres, self.policy_only = kw["board_size"], kw["num_games"], kw["resign_thres"], {}
            self.use_df_feature = kw.get("use_df_feature", False)

    class FakeGame:
        N, resign_thres = 9, 0.0

    def fake_online(**kw):
        got.clear()
        got.update(kw)
        g = FakeGame()
        g.use_df_feature = kw.get("use_df_feature", False)
        return g

    bs = 16
    for mode in ("selfplay", "online"):
        for df in (True, False):
            co, opt = compat.ContextOptions(), compat.GameOptions()
            co.num_games, co.batchsize = 4, bs
            opt.mode, opt.use_df_feature = mode, df
            GC = compat.game_context(co, opt, board_size=9, factories={"selfplay": FakeSelfPlay, "online": fake_online})
            assert got.get("use_df_feature", False) is df and (df or "use_df_feature" not in got), (mode, df)
            p = GC.getParams()
            want = (25, 7, 8) if df else (18, 0, 1)
            assert (p["num_planes"], p["our_stone_plane"], p["opponent_stone_plane"]) == want, (mode, p)
            label = "actor_black" if mode == "selfplay" else "human_actor"
            sm = GC.ctx().allocateSharedMem(GC.ctx().createSharedMemOptions(label, bs), ["s"])
            assert sm["s"].field().sz().vec() == [bs, want[0], 9, 9], (mode, df)


def test_policy_only_colour_in_reference_selfplay():
    """SelfPlay(use_df_feature=True, rng="reference") with white_use_policy_network_only: black searches and
    white moves by MCTSAI_T::actPolicyOnly, both on the DF planes; moves and predicted values equal the
    compiled reference's game threads (RefMctsDf on the same generators)"""
    from elf_b200.selfplay import SelfPlay

    n, G, moves = 9, 2, 20
    need(n)
    opts = dict(num_rollouts=24, num_rollouts_per_batch=4, virtual_loss=1, persistent_tree=1, c_puct=1.5, komi=7.5)
    eps, alpha, cutoff, thres, ratio, move_cutoff = 0.25, 0.3, 6, 0.05, 0.1, 15
    seeds = np.array([771, 772], np.uint64)
    with RefWorker() as w:
        expect, expect_v = w("call", "expected_policy_only_games",
                             (n, seeds, opts, eps, alpha, cutoff, thres, ratio, move_cutoff, moves))

    def actor(batch):
        pi, v = callback(batch["s"].numpy())
        return {"pi": torch.from_numpy(pi), "V": torch.from_numpy(v)}

    gb = emu.emu_batch(G, n)
    mc = df_search(gb, rotation_flip=1, std_sort_ties=1, **opts)
    sp = SelfPlay(actor, num_games=G, board_size=n, board=gb, search=mc, rng="reference", seed=seeds,
                  policy_distri_cutoff=cutoff, resign_thres=thres, never_resign_ratio=ratio, move_cutoff=move_cutoff,
                  root_epsilon=eps, root_alpha=alpha, white_use_policy_network_only=True, use_df_feature=True, **opts)
    got, got_v = [[] for _ in range(G)], [[] for _ in range(G)]
    fin = sp.finish_move

    def logged(info, res=None, chosen=None):
        for g in range(G):
            got[g].append(int(chosen[0][g]))
            got_v[g].append(float(chosen[1][g]))
        return fin(info, res=res, chosen=chosen)

    sp.finish_move = logged
    for _ in range(moves):
        sp.step()
    assert got == expect
    np.testing.assert_allclose(np.array(got_v), np.array(expect_v), rtol=2e-6, atol=1e-7, equal_nan=True)
    assert sp.games_finished >= G
