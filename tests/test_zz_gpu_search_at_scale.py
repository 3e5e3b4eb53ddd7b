"""The self-play search at the benchmark's own size on an H100 (tests/search_scale.py's scenario):
4096 games of 19x19 at 800 rollouts per move and 16,384 games of 9x9 at 400 (BASELINE configs[4]), in
waves of 8 with persistent trees, virtual loss 1, c_puct 1.5 and the default node pool -- the sizes where
a 19x19 part's edge array passes 2^32 bytes and one 4096-game batch's edge slots pass 2^31.  The network
is tests/planenet.py's plane-digest net, a pure function of the leaf planes.

A  the bench's layout (two parts through WavePipeline, f16 NHWC cpad 24, the leaf batch padded to 256)
   against the search restatement on 32 sampled games: equal tables, moves and root values.
B  the same games as one part, float32 NCHW, no padding: every game bitwise equal to A.
C  D4 codes from the reference's own streams, against the compiled reference (19x19).
D  a node pool small enough to prune trees: both layouts agree on every game."""
import gc
import time

import numpy as np
import pytest

import bench
from tests import oracles, planenet
from tests.search_scale import assert_same_tables, check_net, run_scale, sample_games, summary

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

# (board, games, rollouts per move, searched moves): bench.py's default workload and BASELINE configs[4]
SIZES = [(19, bench.GAMES_PER_GPU, bench.ROLLOUTS, 5), (9, 4 * bench.GAMES_PER_GPU, 400, 8)]
PARTS = 2  # bench.py --parts default: two halves interleaved by WavePipeline
_A = {}  # A's tables by board size, for B


def opts(R, **kw):
    return dict(num_rollouts=R, num_rollouts_per_batch=bench.PER_BATCH, virtual_loss=1, persistent_tree=1, c_puct=1.5,
                **kw)


class Peak:
    """the lowest free device memory seen after each move (the node pool is not a torch allocation)"""

    def __init__(self):
        import torch

        self.torch, self.low = torch, None

    def wrap(self, drive):
        def d(searches, net):
            drive(searches, net)
            free, self.total = self.torch.cuda.mem_get_info()
            self.low = free if self.low is None else min(self.low, free)
        return d

    def __str__(self):
        return f"peak device memory in use {(self.total - self.low) / 1e9:.1f} of {self.total / 1e9:.1f} GB"


def room(n, G, R, nodes=0):
    """skip when the node pool (bench.py's estimate: 20.5 B per edge slot) plus 6 GB will not fit"""
    import torch

    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    need = G * (nodes or 2 * R + 256) * (n * n + 1) * 20.5 + (6 << 30)
    if free < need:
        pytest.skip(f"needs about {need / 1e9:.0f} GB of free device memory, {free / 1e9:.0f} GB free")


def pipeline():
    """one move of every part through one WavePipeline, as bench.SelfPlayEngine drives it"""
    from elf_b200.pipeline import WavePipeline

    pipe = []

    def drive(searches, net):
        if not pipe:
            pipe.append(WavePipeline(searches, net))
        pipe[0].search()
    return drive


def one_by_one(searches, net):
    for s in searches:
        s.search(net)


def board(n):
    import elf_b200

    return lambda g: elf_b200.GoBatch(g, board_size=n)


def run_layout(n, G, R, moves, layout, sample=(), nodes=0, **kw):
    """'A': two parts, WavePipeline, f16 NHWC cpad 24, padded to bench.NN_BATCH; 'B': one part, float32
    NCHW, MctsBatch.search with no padding"""
    import elf_b200

    parts, fmt, pad, drive = (PARTS, "f16", bench.NN_BATCH, pipeline()) if layout == "A" else (1, "f32", 0, one_by_one)
    net = planenet.PlaneNet(n, "cuda", batchsize=pad)
    peak = Peak()
    t0 = time.perf_counter()
    r = run_scale(board(n), lambda gb, lo: elf_b200.MctsBatch(gb, feature_format=fmt, cpad=24, rotation_flip=0,
                                                              **opts(R, nodes_per_game=nodes)),
                  peak.wrap(drive), net, n, G, parts, moves, sample=sample, make_state=lambda: oracles.Oracle(n),
                  make_cpu=lambda g: oracles.OracleMcts(n, callback=planenet.callback, **opts(R)),
                  seed=bench.SEED, **kw)
    check_net(net)
    return r, f"; {peak}; {time.perf_counter() - t0:.0f} s"


@pytest.mark.parametrize("n,G,R,moves", SIZES)
def test_a_bench_layout_equals_the_restatement(n, G, R, moves):
    room(n, G, R)
    sample = sample_games(G, PARTS, 32, seed=n)
    r, extra = run_layout(n, G, R, moves, "A", sample=sample)
    print(summary(f"A {n}x{n} G={G} R={R}", r, extra))
    # errors[3] counts trees pruned by the bounded pool (DESIGN §3 (ii)), not an error: this net's priors are
    # peaked (u^8), lines repeat, and a reused subtree can outgrow C - R - 1 slots (1 of 4096 19x19 games by
    # move 5).  Such a game leaves the reference's search; a sampled one would fail below.  B and D check
    # that the pruning is the same in every layout.
    e = r["errors"]
    assert e[0] == 0 and e[1] == 0 and e[2] == 0 and e[3] <= G // 256, e
    assert r["compared"] >= (moves - 1) * len(sample) and r["exact"] == r["compared"]
    assert (r["total_visits"][-1] > R).mean() > 0.5  # the trees were reused across moves
    _A[n] = r


@pytest.mark.parametrize("n,G,R,moves", SIZES)
def test_b_one_float32_part_equals_the_bench_layout(n, G, R, moves):
    if n not in _A:
        pytest.skip("needs the tables of test_a_bench_layout_equals_the_restatement in the same session")
    room(n, G, R)
    r, extra = run_layout(n, G, R, moves, "B")
    print(summary(f"B {n}x{n} G={G} R={R}", r, extra))
    np.testing.assert_array_equal(r["errors"], _A[n]["errors"])
    assert_same_tables(_A[n], r, f"{n}x{n}: one float32 part vs two f16 parts")


@pytest.mark.skipif(not oracles.have_ref(19), reason="compiled reference (oracle/_ref) not available")
def test_c_reference_streams_against_the_compiled_reference():
    """the bench runs with rotation_flip=1: every evaluated leaf is written under a D4 code.  Here the codes
    come from the reference's own generators (RefStream, a seed per game, init_actor(0)), so the compiled
    reference (RefMcts seeded as init_ai seeds it) draws the same ones; equal fp priors are ordered by
    std::sort as in the reference (std_sort_ties).  Bar as in test_gpu_mcts.py: every edge within +-1, the
    same move where a table is exact."""
    import elf_b200
    from elf_b200.refstream import RefStream

    n, G, R, moves = SIZES[0]
    room(n, G, R)
    seeds = np.arange(G, dtype=np.uint64) + np.uint64(bench.SEED)

    def search(gb, lo):
        mc = elf_b200.MctsBatch(gb, feature_format="f16", cpad=24, rotation_flip=1, std_sort_ties=1, **opts(R))
        rs = RefStream(gb.num_games, n, seeds[lo: lo + gb.num_games])
        rs.init_actor(0)
        mc.attach_ref_stream(rs, 0)
        return mc

    def ref_search(g):
        seed = oracles.RefRng(n, int(seeds[g])).next()
        return oracles.RefMcts(n, callback=planenet.callback, rotation_flip=1, seed=seed, **opts(R))

    net = planenet.PlaneNet(n, "cuda", batchsize=bench.NN_BATCH)
    peak = Peak()
    t0 = time.perf_counter()
    sample = sample_games(G, PARTS, 16, seed=3)
    r = run_scale(board(n), search, peak.wrap(pipeline()), net, n, G, PARTS, moves, sample=sample,
                  make_state=lambda: oracles.Ref(n), make_cpu=ref_search, tol=1, seed=bench.SEED)
    check_net(net)
    print(summary(f"C {n}x{n} G={G} R={R} reference streams", r, f"; {peak}; {time.perf_counter() - t0:.0f} s"))
    e = r["errors"]  # errors[3]: pruned trees, as in test_a
    assert e[0] == 0 and e[1] == 0 and e[2] == 0 and e[3] <= G // 256, e
    assert r["compared"] >= (moves - 1) * len(sample)


@pytest.mark.parametrize("n,G,R,moves", SIZES)
def test_d_pruned_trees_agree_between_layouts(n, G, R, moves):
    """a node pool of R + 64 slots per game: at the start of a move a reused tree must be pruned
    (DESIGN §3 (ii), no reference); both layouts prune the same games the same way"""
    nodes = R + 64
    room(n, G, R, nodes)
    a, ea = run_layout(n, G, R, moves, "A", nodes=nodes)
    print(summary(f"D {n}x{n} G={G} R={R} nodes_per_game={nodes}, layout A", a, ea))
    b, eb = run_layout(n, G, R, moves, "B", nodes=nodes)
    print(summary(f"D {n}x{n} G={G} R={R} nodes_per_game={nodes}, layout B", b, eb))
    for e in (a["errors"], b["errors"]):
        assert e[3] > 0 and e[0] == 0 and e[1] == 0 and e[2] == 0, e
    assert_same_tables(a, b, f"{n}x{n} pruned: one float32 part vs two f16 parts")
