"""tests/search_scale.py's scenario on the SIMT emulator build of the kernel sources, at a small size:
the bench's layout (two parts searched in turn, f16 NHWC cpad 24 leaf planes, the leaf batch padded to
the network's batch size) and the other one (one part, float32 NCHW, no padding), each against the
search restatement on the same plane-digest net, and bitwise against each other.  The GPU run at the
bench's own size is tests/test_zz_gpu_search_at_scale.py."""
import numpy as np
import pytest

from tests import oracles, planenet
from tests.search_scale import assert_same_tables, check_net, padded_search, run_scale, sample_games, summary

pytestmark = pytest.mark.timeout(900)


@pytest.fixture(scope="module")
def emu():
    from tests import emu as E

    try:
        E.emu_lib()
    except Exception as e:  # no g++ / ucontext: the emulator is a convenience, not a requirement
        pytest.skip(f"SIMT emulator build unavailable: {e}")
    return E


# (n, G, rollouts, moves, network batch size): 9x9 with G = 9 fills three warps of three games, the part
# of 5 games leaves a warp with one game
@pytest.mark.parametrize("n,G,R,moves,pad", [(19, 6, 64, 5, 16), (9, 9, 64, 8, 16)])
def test_search_scale_on_the_emulator(emu, oracle_lib, n, G, R, moves, pad):
    opts = dict(num_rollouts=R, num_rollouts_per_batch=8, virtual_loss=1, persistent_tree=1, c_puct=1.5)
    sample = sample_games(G, 2, count=G)

    def run(parts, fmt, batchsize):
        net = planenet.PlaneNet(n, "cpu", batchsize=batchsize)
        r = run_scale(lambda g: emu.emu_batch(g, n),
                      lambda gb, lo: emu.EmuSearch(gb, feature_format=fmt, cpad=24, rotation_flip=0, **opts),
                      padded_search, net, n, G, parts, moves, sample=sample,
                      make_state=lambda: oracles.Oracle(n, oracle_lib),
                      make_cpu=lambda g: oracles.OracleMcts(n, lib=oracle_lib, callback=planenet.callback, **opts))
        check_net(net)
        assert (r["errors"] == 0).all(), r["errors"]
        assert r["compared"] == moves * len(sample) and r["exact"] == r["compared"]
        print(summary(f"emu {n}x{n} G={G} parts={parts} {fmt}", r))
        return r

    a = run(2, "f16", pad)
    b = run(1, "f32", 0)
    assert_same_tables(a, b, "two padded f16 parts vs one f32 part")
    assert (a["total_visits"][1:] > R).any()  # the trees were reused across moves
