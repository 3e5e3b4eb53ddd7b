"""Copying games between batches on the H100: the reference parity of tests/test_gather.py through the same
run functions, full-size branch batches (4 branches per source game) played on and restarted from a
position pool against cloned reference states, a CUDA graph of step -> gather -> step over two contexts
against the same loop run eagerly, and a search with a 20x256 network from copied positions."""
import numpy as np
import pytest
import torch

from tests import oracles
from tests.test_env import KOMI
from tests.test_gather import (need_ref, random_moves, ref_clone, run_copies_played_on, run_copy_equals_reference,
                               run_env_load, run_search_on_copies, run_superko_record_copied)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

K = 4  # branches per source game


def _gobatch(G, n):
    import elf_b200

    return elf_b200.GoBatch(G, board_size=n)


def make_env(G, n, **kw):
    from elf_b200.env import GoEnv

    return GoEnv.create(G, board_size=n, **kw)


make_env.batch = _gobatch


@pytest.mark.parametrize("n", [9, 19])
def test_copy_equals_reference_copy(n):
    need_ref(n)
    run_copy_equals_reference(_gobatch, n, seed=n)


@pytest.mark.parametrize("n", [9, 19])
def test_copies_stay_equal_when_played_on(n):
    need_ref(n)
    run_copies_played_on(make_env, n, seed=2 * n)


def test_copied_superko_record():
    need_ref(9)
    run_superko_record_copied(make_env)


def test_search_on_copies_equals_search_on_originals():
    import elf_b200

    need_ref(9)
    run_search_on_copies(_gobatch, elf_b200.MctsBatch)


def test_env_load():
    need_ref(9)
    run_env_load(make_env)


def _policy(legal, counter, gen, seed):
    """random_legal_actions with a pass one time in eight, so that games also end by two passes"""
    from elf_b200.env import random_legal_actions

    a = random_legal_actions(legal, counter, seed=seed)
    return torch.where(torch.rand(a.shape, generator=gen, device=a.device) < 0.125, legal.shape[1] - 1, a).to(torch.int32)


def _replay_refs(acts, done, G, n, sample):
    """reference states of the sampled games after their logged actions (fresh where a game ended)"""
    refs = {}
    for g in sample:
        r = oracles.Ref(n)
        for t in range(acts.shape[0]):
            if acts[t, g] >= 0:
                r.forward(int(acts[t, g]))
            assert r.terminated() == bool(done[t, g]), (g, t)
            if done[t, g]:
                r = oracles.Ref(n)
        refs[g] = r
    return refs


@pytest.mark.parametrize("n,G", [(19, 4096), (9, 12288)])
def test_branches_at_scale(n, G):
    """G source games played by the seeded device policy to a spread of plies (every game stops at its own
    ply); copied into K * G branch slots (index arange(G).repeat_interleave(K)): hash, info, legal and AGZ
    planes equal their source's, compared on the device.  Then 64 plies of every branch under the policy,
    finished games restarted from a pool of positions built with GoBatch.replay (GoEnv.load with
    torch.where(done, pick, -1)); a seeded sample of 256 branches is compared every ply with cloned reference
    states: ok, done, value bit for bit, legal and info, and the hash at the end."""
    need_ref(n)
    dev = torch.device("cuda", 0)
    P, A = n * n, n * n + 1
    T0 = 150 if n == 19 else 60
    src = make_env(G, n, features="f16")
    obs = src.reset()
    counter = torch.zeros(1, dtype=torch.int64, device=dev)
    gen = torch.Generator(device=dev)
    gen.manual_seed(n)
    stop = torch.randint(T0 // 2, T0 + 1, (G,), generator=gen, device=dev)
    log_a = torch.empty((T0, G), dtype=torch.int32, device=dev)
    log_d = torch.empty((T0, G), dtype=torch.uint8, device=dev)
    for t in range(T0):
        a = torch.where(stop > t, _policy(obs["legal"], counter, gen, seed=1), -1).to(torch.int32)
        log_a[t] = a
        obs = src.step(a)
        log_d[t] = obs["done"]
    idx = torch.arange(G, device=dev, dtype=torch.int32).repeat_interleave(K)
    br = make_env(K * G, n, features="f16")
    bobs = br.load(src, idx)
    il = idx.long()
    for k in ("legal", "info", "planes"):
        assert torch.equal(bobs[k], obs[k][il]), k
    assert (br.board.getHashCode() == src.board.getHashCode()[idx.cpu().numpy()]).all()
    assert not bobs["ok"].any() and not bobs["done"].any()
    plies = src.board.getPly()
    assert plies.min() < plies.max() - 20  # a spread of plies
    # the position pool
    rng = np.random.default_rng(n)
    pool_moves = [random_moves(oracles.Ref(n), rng, int(rng.integers(0, P))) for _ in range(64)]
    pool = _gobatch(len(pool_moves), n)
    pool.replay(pool_moves)
    pick = torch.randint(0, len(pool_moves), (64, K * G), generator=gen, device=dev, dtype=torch.int32)
    sample = np.sort(rng.choice(K * G, 256, replace=False))
    sd = torch.from_numpy(sample).to(dev)
    T = 64
    c2 = torch.zeros(1, dtype=torch.int64, device=dev)
    la = torch.empty((T, K * G), dtype=torch.int32, device=dev)
    lok, ldone = torch.empty((T, K * G), dtype=torch.uint8, device=dev), torch.empty((T, K * G), dtype=torch.uint8, device=dev)
    lval = torch.empty((T, K * G), dtype=torch.float32, device=dev)
    llegal = torch.empty((T, 256, A), dtype=torch.bool, device=dev)
    linfo = torch.empty((T, 256, 12), dtype=torch.int32, device=dev)
    for t in range(T):
        a = _policy(bobs["legal"], c2, gen, seed=2)
        la[t] = a
        bobs = br.step(a)
        lok[t], ldone[t], lval[t] = bobs["ok"], bobs["done"], bobs["value"]
        bobs = br.load(pool, torch.where(bobs["done"].bool(), pick[t], -1).to(torch.int32))
        llegal[t], linfo[t] = bobs["legal"][sd], bobs["info"][sd]
    acts0, done0 = log_a.cpu().numpy(), log_d.cpu().numpy()
    acts, ok, done, val = la.cpu().numpy(), lok.cpu().numpy(), ldone.cpu().numpy(), lval.cpu().numpy()
    legal, info, pk = llegal.cpu().numpy(), linfo.cpu().numpy(), pick.cpu().numpy()
    h = br.board.getHashCode()
    assert done.sum() > 0
    srcs = _replay_refs(acts0, done0, G, n, sorted({int(s) // K for s in sample}))
    pool_refs = []
    for m in pool_moves:
        r = oracles.Ref(n)
        for a in m:
            r.forward(a)
        pool_refs.append(r)
    restarts = 0
    for j, g in enumerate(sample):
        r = ref_clone(srcs[g // K])
        for t in range(T):
            assert r.forward(int(acts[t, g])) == bool(ok[t, g]), (g, t)
            assert r.terminated() == bool(done[t, g]), (g, t)
            if done[t, g]:
                assert val[t, g].tobytes() == np.float32(r.evaluate(KOMI)).tobytes(), (g, t)
                r = ref_clone(pool_refs[pk[t, g]])
                restarts += 1
            np.testing.assert_array_equal(legal[t, j, :P], r.legal().astype(bool), err_msg=f"legal {g} {t}")
            ri = r.info()
            ri[8] = 0
            np.testing.assert_array_equal(info[t, j], ri, err_msg=f"info {g} {t}")
        assert int(h[g]) == r.hash(), g
    assert restarts > 0
    br.close()
    src.close()
    pool.close()


def test_cuda_graph_of_step_gather_step_equals_eager():
    """8 rounds of  policy -> source GoEnv.step -> GoEnv.load(source, index) -> policy -> branch
    GoEnv.step  (fp16 planes) over two contexts, captured once and replayed twice; the same loop run eagerly
    from the same start on two other contexts: hashes, ok, done, value, legal, info and planes of both
    contexts are bitwise equal after each replay"""
    from elf_b200.env import random_legal_actions

    n, G = 19, 1024
    dev = torch.device("cuda", 0)
    idx = torch.arange(G, device=dev, dtype=torch.int32).repeat_interleave(K)
    idx = torch.where(torch.arange(K * G, device=dev) % 5 == 3, -1, idx).to(torch.int32)  # some branches keep their game
    twins = []
    for _ in range(2):
        s, b = make_env(G, n, features="f16"), make_env(K * G, n, features="f16")
        so, bo = s.reset(), b.reset()
        bo = b.load(s, idx)  # also creates the gather's events outside the capture
        twins.append([s, b, so, bo, torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int64, device=dev)])
    random_legal_actions(torch.ones((K * G, n * n + 1), dtype=torch.bool, device=dev), torch.zeros(1, dtype=torch.int64, device=dev))
    torch.cuda.synchronize()

    def rounds(tw):
        s, b, so, bo, c1, c2 = tw
        for _ in range(8):
            so = s.step(random_legal_actions(so["legal"], c1, seed=1))
            bo = b.load(s, idx)
            bo = b.step(random_legal_actions(bo["legal"], c2, seed=2))
        tw[2], tw[3] = so, bo

    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        rounds(twins[0])
    for rep in range(2):
        graph.replay()
        rounds(twins[1])
        torch.cuda.synchronize()
        for i in (0, 1):  # the source, then the branches
            eg, ee = twins[0][i], twins[1][i]
            assert (eg.board.getHashCode() == ee.board.getHashCode()).all(), (rep, i)
            for k in ("ok", "done", "value", "legal", "info", "planes"):
                assert torch.equal(eg.obs[k], ee.obs[k]), (rep, i, k)
    assert (twins[0][1].board.getPly() > 10).any()
    for tw in twins:
        tw[0].close()
        tw[1].close()


def test_search_on_copies_with_a_network():
    """MctsBatch with a random-init 20x256 network on 8 copied 19x19 positions (copies in another batch,
    same slots) equals the search on the originals: root visits and chosen moves"""
    import elf_b200
    from elf_b200.model import Actor, PolicyValueNet

    n, G = 19, 8
    torch.manual_seed(0)
    net = PolicyValueNet(n, num_block=20, dim=256).cuda()
    rng = np.random.default_rng(4)
    lists = [random_moves(oracles.Ref(n), rng, int(rng.integers(20, 200))) for _ in range(G)]
    src = _gobatch(G, n)
    src.replay(lists)
    dst = _gobatch(G, n)
    dst.forward(np.full(G, 60, np.int32))
    dst.gather(src, torch.arange(G, dtype=torch.int32, device="cuda"))
    res = []
    for gb in (src, dst):
        mc = elf_b200.MctsBatch(gb, rotation_flip=0, num_rollouts=200, num_rollouts_per_batch=16, virtual_loss=1,
                                persistent_tree=1, c_puct=1.5)
        res.append(mc.act(Actor(net, batchsize=64)))
        assert (mc.errors() == 0).all()
        mc.close()
    np.testing.assert_array_equal(res[0]["visits"], res[1]["visits"])
    np.testing.assert_array_equal(res[0]["best_action"], res[1]["best_action"])
    assert (src.getHashCode() == dst.getHashCode()).all()
    src.close()
    dst.close()
