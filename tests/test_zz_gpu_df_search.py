"""The search on the DarkForest planes (GameOptions::use_df_feature) on an H100: k_leaf_features_df behind
MctsBatch(feature_format="df") against the compiled reference's search on BoardFeature::extract's planes
(tests/df_search.py), at small sizes and at the benchmark's, and GPU self-play with a 25-plane network."""
import time

import numpy as np
import pytest

from tests import oracles
from tests.df_search import DfNet, RefWorker, have_df_ref, ko_line, random_lines, run_df_search

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

OPTS = dict(num_rollouts=64, num_rollouts_per_batch=8, virtual_loss=1, persistent_tree=1, c_puct=1.5)


def need(n):
    if not have_df_ref(n):
        pytest.skip("compiled reference (oracle/_ref) not available")


def make(G, n, flip=0, seeds=None, **opts):
    import elf_b200
    from elf_b200.refstream import RefStream

    gb = elf_b200.GoBatch(G, board_size=n)
    mc = elf_b200.MctsBatch(gb, feature_format="df", rotation_flip=flip, std_sort_ties=flip, **opts)
    if flip:
        rs = RefStream(G, n, np.asarray(seeds, np.uint64))
        rs.init_actor(0)
        mc.attach_ref_stream(rs, 0)
    return gb, mc


HANDICAP = lambda n, G: [[a * n + b for a, b in ((2, 2), (n - 3, n - 3), (2, n - 3), (n - 3, 2))]] * G  # noqa: E731
SCENARIOS = {
    "fresh_after_captures": (lambda n, G: random_lines(n, G, 40 if n == 9 else 90, 21, captures=True), None, 1),
    "persistent_5_moves": (lambda n, G: random_lines(n, G, 10, 22), None, 5),
    "ko_fight": (lambda n, G: [ko_line(n)] * G, None, 3),  # with ko_callback: the fight is forced
    "handicap_ply1": (None, HANDICAP, 3),
    "near_ply_cap": (lambda n, G: random_lines(n, G, 2 * n * n - 20, 23), None, 3),
}


@pytest.mark.parametrize("flip", [0, 1])
@pytest.mark.parametrize("scenario", sorted(SCENARIOS))
@pytest.mark.parametrize("n", [9, 19])
def test_search_equals_reference_on_device(n, scenario, flip):
    need(n)
    G = 2 if scenario == "near_ply_cap" else 4
    lines_f, hcap_f, moves = SCENARIOS[scenario]
    seeds = [20261017 + g for g in range(G)] if flip else None
    gb, mc = make(G, n, flip, seeds, **OPTS)
    try:
        run_df_search(gb, mc, n, OPTS, moves, lines=lines_f(n, G) if lines_f else None,
                      handicap=hcap_f(n, G) if hcap_f else None, seeds=seeds,
                      net_name="ko" if scenario == "ko_fight" else "plain",
                      plane_check=(scenario == "ko_fight" and flip == 0))
    finally:
        mc.close()
        gb.close()


@pytest.mark.parametrize("n,G,R,moves", [(19, 4096, 800, 3), (9, 16384, 400, 3)])
def test_bench_size_against_reference(n, G, R, moves):
    """the benchmark's size on the DF planes: two parts through WavePipeline, the torch twin of the digest net
    padded to 256, reference D4 streams; 16 sampled games per size against the compiled reference"""
    need(n)
    import torch

    import elf_b200
    from elf_b200.pipeline import WavePipeline
    from elf_b200.refstream import RefStream
    from tests.search_scale import run_scale, sample_games, summary

    opts = dict(num_rollouts=R, num_rollouts_per_batch=8, virtual_loss=1, persistent_tree=1, c_puct=1.5)
    seeds = np.arange(G, dtype=np.uint64) + np.uint64(20260922)

    def search(gb, lo):
        mc = elf_b200.MctsBatch(gb, feature_format="df", rotation_flip=1, std_sort_ties=1, **opts)
        rs = RefStream(gb.num_games, n, seeds[lo: lo + gb.num_games])
        rs.init_actor(0)
        mc.attach_ref_stream(rs, 0)
        return mc

    w = RefWorker()  # the reference's states and searches in a child process

    def ref_search(g):
        return w.search(n, rotation_flip=1, seed=w("call", "actor_seed", (n, int(seeds[g]))), **opts)

    pipe, low = [], [None]

    def drive(searches, net):
        if not pipe:
            pipe.append(WavePipeline(searches, net))
        pipe[0].search()
        free, total = torch.cuda.mem_get_info()
        low[0] = free if low[0] is None else min(low[0], free)
        low.append(total)

    net = DfNet(n, "cuda", batchsize=256)
    t0 = time.perf_counter()
    try:
        r = run_scale(lambda g: elf_b200.GoBatch(g, board_size=n), search, drive, net, n, G, 2, moves,
                      sample=sample_games(G, 2, 16, seed=n), make_state=lambda: w.state(n), make_cpu=ref_search, tol=1,
                      seed=20260922)
    finally:
        w.close()
    total = low[-1]
    print(summary(f"DF {n}x{n} G={G} R={R} reference streams", r,
                  f"; peak device memory in use {(total - low[0]) / 1e9:.1f} of {total / 1e9:.1f} GB; "
                  f"{time.perf_counter() - t0:.0f} s"))
    e = r["errors"]
    assert e[0] == 0 and e[1] == 0 and e[2] == 0 and e[3] <= G // 256, e
    assert r["compared"] >= (moves - 1) * 16 and net.calls > 0


def test_selfplay_df_network_records_accepted_by_reference():
    """SelfPlay(use_df_feature=True) with a 25-plane PolicyValueNet behind FusedActor(cpad=32): 64 games; the
    records go through the reference's Record::createFromJson"""
    import json

    import torch

    import elf_b200
    from elf_b200 import record
    from elf_b200.model import FusedActor, PolicyValueNet

    n, G = 9, 64
    if not oracles.have_ref(n):
        pytest.skip("oracle/_ref not built")
    torch.manual_seed(3)
    net = PolicyValueNet(n, num_planes=25, num_block=1, dim=16).cuda().eval()
    actor = FusedActor(net, batchsize=64, dtype=torch.float16, cuda_graph=True, cpad=32)
    seen = []
    inner = actor.__call__

    class Spy:
        batchsize = actor.batchsize

        def __call__(self, batch):
            seen.append(tuple(batch["s"].shape[1:]))
            return inner(batch)

    sp = elf_b200.selfplay.SelfPlay(Spy(), num_games=G, board_size=n, policy_distri_cutoff=4, num_rollouts=16,
                                    num_rollouts_per_batch=4, move_cutoff=12, seed=5, record_games=True,
                                    resign_thres=0.0, use_df_feature=True, white_use_policy_network_only=True)
    assert sp.mcts.feature_format == "df"
    while sp.games_finished < G:
        sp.step()
    assert seen and all(s == (25, n, n) for s in seen)
    recs = sp.records
    assert len(recs) >= G
    assert oracles.ref_record_batch_count(record.dumps(recs), n) == len(recs)
    for rec in recs:
        assert oracles.ref_record_roundtrip(json.dumps(rec), n) is not None
    sp.close()
    with pytest.raises(ValueError):
        elf_b200.selfplay.SelfPlay(Spy(), num_games=2, board_size=n, use_df_feature=True, feature_format="bf16")
