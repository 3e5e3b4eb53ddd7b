"""The search on the DarkForest planes (GameOptions::use_df_feature) against the compiled reference (test
infrastructure only).

* ``digest_np`` / ``DfNet``: a deterministic test network keyed by the leaf's 25 planes.  The DF history
  and distance planes are not 0/1, so the digest reads the float32 BIT PATTERNS: every entry's pattern is
  split into its low and high 16 bits, each dotted with fixed 31-bit weights as an int64 sum (products
  < 2^47, 25*361 of them: no overflow, any summation order gives the same integer), and the key
  ``s_lo + 2 * s_hi`` is answered by ``oracles.fakenet``.  ``callback`` is the numpy twin (the reference's
  callback), ``DfNet`` the torch twin on the tensors' device.
* ``RefMctsDf``: oracle/ref_mcts_df_shim.cc (``ref_mcts_new_df``), the reference search whose network sees
  BoardFeature::extract's planes, on states of ``oracles.Ref``.
* ``RefWorker``: the reference states and searches live in a child process.  The reference's search sums edge
  rewards in the order of its nodes' heap addresses, so its visit tables can depend on what the process
  allocated before; in a fresh child they do not depend on earlier tests, and the tests' own process is
  left as it was.
* ``run_df_search``: our search and the reference's, move for move, on prepared positions."""
import ctypes
import os

import numpy as np

from tests import oracles

vp = ctypes.c_void_p
PLANES = 25


def df_ref_path(n):
    return os.path.join(oracles.ORACLE_DIR, "_ref", f"libref_mcts_df{n}.so")


def have_df_ref(n):
    return oracles.have_ref(n) and os.path.exists(df_ref_path(n))


def weights(n):
    """int64 [25, n, n]: 31-bit weights by (plane, row, column)"""
    i = np.arange(PLANES * n * n, dtype=np.uint64) + np.uint64((n << 40) | 0xDF)
    return (oracles._splitmix64(i) >> np.uint64(33)).astype(np.int64).reshape(PLANES, n, n)


def digest_np(planes):
    """uint64 [m]: the digest of float32 planes [m, 25, n, n]"""
    x = np.ascontiguousarray(planes, dtype=np.float32)
    m, C, n, _ = x.shape
    assert C == PLANES, x.shape
    b = x.view(np.uint32).reshape(m, -1).astype(np.int64)
    W = weights(n).reshape(-1)
    s_lo, s_hi = (b & 0xFFFF) @ W, (b >> 16) @ W
    return (s_lo + 2 * s_hi).astype(np.uint64)


def callback(feats, hashes=None):
    """``callback(feats [m,25,n,n] float32, hashes)`` of RefMctsDf: (pi [m,N*N+1], v [m])"""
    n = feats.shape[-1]
    return oracles.fakenet(digest_np(feats), n * n + 1)


class DfNet:
    """the torch twin: ``net(batch) -> {"pi", "V"}`` from ``batch["s"]`` float32 [m,25,n,n] on its device, no
    host synchronisation.  ``batchsize``: the search pads its leaf batch to a multiple of it."""

    def __init__(self, n, device, batchsize=0, chunk=2048):
        import torch

        self.torch, self.n, self.batchsize, self.chunk = torch, n, batchsize, chunk
        self.W = torch.from_numpy(weights(n)).to(device)
        self.calls = 0

    def digest(self, x):
        torch = self.torch
        out = torch.empty(x.shape[0], dtype=torch.int64, device=x.device)
        for lo in range(0, x.shape[0], self.chunk):
            b = x[lo: lo + self.chunk].contiguous().view(torch.int32).to(torch.int64)
            s_lo = ((b & 0xFFFF) * self.W).flatten(1).sum(1)
            s_hi = ((b >> 16) * self.W).flatten(1).sum(1)
            out[lo: lo + self.chunk] = s_lo + 2 * s_hi
        return out

    def __call__(self, batch):
        from tests.planenet import fakenet_torch

        self.calls += 1
        x = batch["s"]
        assert x.dtype == self.torch.float32 and tuple(x.shape[1:]) == (PLANES, self.n, self.n), tuple(x.shape)
        pi, v = fakenet_torch(self.digest(x), self.n * self.n + 1)
        return {"pi": pi, "V": v}


class RefMctsDf:
    """the reference search on the DarkForest planes; ``act`` as ``oracles.RefMcts.act``"""

    def __init__(self, n, callback, num_rollouts=200, num_rollouts_per_batch=8, virtual_loss=1, persistent_tree=1,
                 use_prior=1, unexplored_q_zero=0, root_unexplored_q_zero=0, ply_pass_enabled=0,
                 remove_pass_if_dangerous=1, seed=7, c_puct=1.5, komi=7.5, root_epsilon=0.0, root_alpha=0.0,
                 rotation_flip=0, **_):
        oracles.load_ref(n)  # the board library first: the shim links against this very instance
        self.L = L = ctypes.CDLL(df_ref_path(n))
        self.n = n
        L.ref_mcts_new_df.restype = vp
        L.ref_mcts_new_df.argtypes = [vp, vp, vp, ctypes.c_int, ctypes.c_uint32]
        L.ref_mcts_df_act.argtypes = [vp, vp, ctypes.c_int] + [vp] * 6
        L.ref_mcts_df_free.argtypes = [vp]
        L.ref_mcts_df_num_evals.restype = ctypes.c_long
        L.ref_mcts_df_num_evals.argtypes = [vp]
        iopts = np.array([num_rollouts, num_rollouts_per_batch, virtual_loss, persistent_tree, use_prior,
                          unexplored_q_zero, root_unexplored_q_zero, ply_pass_enabled, remove_pass_if_dangerous,
                          int(seed) & 0x7FFFFFFF, 1], np.int32)
        fopts = np.array([c_puct, komi, root_epsilon, root_alpha], np.float32)
        CB = ctypes.CFUNCTYPE(None, ctypes.c_int, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint64),
                              ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float))
        P1 = n * n + 1

        def tramp(cnt, feats, hashes, pi, v):
            f = np.ctypeslib.as_array(feats, shape=(cnt, PLANES, n, n))
            h = np.ctypeslib.as_array(hashes, shape=(cnt,))
            p, val = callback(f, h)
            np.ctypeslib.as_array(pi, shape=(cnt, P1))[:] = p
            np.ctypeslib.as_array(v, shape=(cnt,))[:] = val

        self._cb = CB(tramp)
        self.m = L.ref_mcts_new_df(iopts.ctypes.data, fopts.ctypes.data, ctypes.cast(self._cb, vp), int(rotation_flip),
                                   int(seed) & 0xFFFFFFFF)

    def act(self, ref_state, policy_only=False):
        P1 = self.n * self.n + 1
        vis, w, pr = np.zeros(P1, np.int32), np.zeros(P1, np.float32), np.zeros(P1, np.float32)
        rv, bq, tv = ctypes.c_float(), ctypes.c_float(), ctypes.c_int32()
        a = self.L.ref_mcts_df_act(self.m, ref_state.p, int(bool(policy_only)), vis.ctypes.data, w.ctypes.data,
                                   pr.ctypes.data, ctypes.byref(rv), ctypes.byref(bq), ctypes.byref(tv))
        return {"best_action": int(a), "visits": vis, "wsum": w, "prior": pr, "root_value": rv.value,
                "best_q": bq.value, "total_visits": tv.value}

    def num_evals(self):
        return int(self.L.ref_mcts_df_num_evals(self.m))

    def sample(self, rng):
        """mcts_make_diverse_move's sampling on the game thread's generator (an oracles.RefRng)"""
        self.L.ref_mcts_df_sample.argtypes = [vp, vp]
        return int(self.L.ref_mcts_df_sample(self.m, rng.p))

    def end_game(self, ref_state):
        """MCTSAI_T::endGame: the tree is reset"""
        self.L.ref_mcts_df_end_game.argtypes = [vp, vp]
        self.L.ref_mcts_df_end_game(self.m, ref_state.p)

    def __del__(self):
        if getattr(self, "m", None):
            self.L.ref_mcts_df_free(self.m)
            self.m = None


# ---- the reference in a child process ------------------------------------------------------------------
NETS = {"plain": lambda n: callback, "ko": lambda n: ko_callback(n)}


def _worker_main(conn):
    objs, recorded, ids = {}, {}, iter(range(1 << 30))

    def recording(net):
        def cb(feats, hashes):
            for f, h in zip(feats, hashes):
                recorded.setdefault(int(h), []).append(f.copy())
            return net(feats, hashes)
        return cb

    while True:
        msg = conn.recv()
        if msg is None:
            break
        op, args = msg
        try:
            if op == "new_state":
                k = next(ids)
                objs[k] = oracles.Ref(args[0])
                r = k
            elif op == "new_search":
                n, net, record, kw = args
                cb = NETS[net](n)
                k = next(ids)
                objs[k] = RefMctsDf(n, recording(cb) if record else cb, **kw)
                r = k
            elif op == "act":
                sid, stid, policy_only = args
                r = objs[sid].act(objs[stid], policy_only=policy_only)
            elif op == "method":
                k, name, margs = args
                r = getattr(objs[k], name)(*margs)
            elif op == "place_handicap":
                from tests.test_handicap import ref_place_handicap

                r = ref_place_handicap(objs[args[0]], args[1])
            elif op == "recorded":
                r = dict(recorded)
                recorded.clear()
            elif op == "call":  # a module-level function of this module
                r = globals()[args[0]](*args[1])
            else:
                raise ValueError(op)
            conn.send((True, r))
        except Exception as e:  # noqa: BLE001 -- handed to the caller
            conn.send((False, f"{type(e).__name__}: {e}"))


class RefWorker:
    """a child process (spawn: a fresh heap, no device) holding reference states and RefMctsDf searches"""

    def __init__(self):
        import multiprocessing as mp

        ctx = mp.get_context("spawn")
        self.conn, child = ctx.Pipe()
        self.proc = ctx.Process(target=_worker_main, args=(child,), daemon=True)
        self.proc.start()
        child.close()

    def __call__(self, op, *args):
        self.conn.send((op, args))
        ok, r = self.conn.recv()
        if not ok:
            raise AssertionError(f"reference worker: {r}")
        return r

    def close(self):
        if self.proc is not None:
            self.conn.send(None)
            self.proc.join(60)
            self.conn.close()
            self.proc = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def state(self, n):
        return RefStateProxy(self, n)

    def search(self, n, net="plain", record=False, **kw):
        return RefSearchProxy(self, n, net, record, kw)


class RefStateProxy:
    """an oracles.Ref in the worker: forward / terminated / info / stones"""

    def __init__(self, w, n):
        self.w, self.n, self.k = w, n, w("new_state", n)

    def __getattr__(self, name):
        if name in ("forward", "terminated", "info", "stones", "hash"):
            return lambda *a: self.w("method", self.k, name, tuple(int(x) for x in a))
        raise AttributeError(name)


class RefSearchProxy:
    """a RefMctsDf in the worker: act / num_evals"""

    def __init__(self, w, n, net, record, kw):
        self.w, self.n, self.k = w, n, w("new_search", n, net, record, kw)

    def act(self, state, policy_only=False):
        return self.w("act", self.k, state.k, bool(policy_only))

    def num_evals(self):
        return self.w("method", self.k, "num_evals", ())


def actor_seed(n, seed):
    """the seed init_ai gives an actor: the first draw of a game thread's generator seeded with ``seed``"""
    return oracles.RefRng(n, int(seed)).next()


def expected_policy_only_games(n, seeds, opts, eps, alpha, cutoff, thres, ratio, move_cutoff, moves):
    """the reference's game threads with white_use_policy_network_only on the DF planes (run in a RefWorker):
    per seed the moves played and the predicted values, across game ends"""
    expect, expect_v = [], []
    for s in seeds:
        g = oracles.RefRng(n, int(s))
        ai = RefMctsDf(n, callback, root_epsilon=eps, root_alpha=alpha, rotation_flip=1, seed=g.next(), **opts)
        rc = oracles.RefResign(n, thres, ratio)
        st = oracles.Ref(n)
        played, values = [], []
        for _ in range(moves):
            ply, nxt = int(st.info()[0]), int(st.info()[1])
            if nxt == 2:
                r = ai.act(st, policy_only=True)
                a = r["best_action"]
            else:
                r = ai.act(st)
                a = ai.sample(g) if ply <= cutoff else r["best_action"]
            rc.check(r["best_q"], nxt, g)
            assert st.forward(int(a))
            played.append(int(a))
            values.append(float(r["best_q"]))
            if st.info()[9] or int(st.info()[0]) >= move_cutoff:
                ai.end_game(st)
                st = oracles.Ref(n)
                rc.reset()
        expect.append(played)
        expect_v.append(values)
    return expect, expect_v


# ---- positions ----------------------------------------------------------------------------------------
def random_lines(n, G, plies, seed, captures=False):
    """per game ``plies`` uniformly random legal non-pass moves on a host state (a game that ends or
    runs out of points is drawn again); ``captures``: only games where a stone was captured"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < G:
        r = oracles.Oracle(n)
        line, ok = [], True
        for _ in range(plies):
            pts = np.flatnonzero(r.legal())
            if len(pts) == 0:
                ok = False
                break
            a = int(rng.choice(pts))
            assert r.forward(a)
            line.append(a)
        stones = int((r.stones() != 0).sum())
        if ok and not r.terminated() and (not captures or stones < plies):
            out.append(line)
    return out


def ko_line(n):
    """a simple ko ready to be taken: black to move captures at (4,5), white may retake (4,4) later
    (actions x*N+y); the points around it are the only stones"""
    a = lambda x, y: x * n + y  # noqa: E731
    return [a(3, 4), a(3, 5), a(4, 3), a(4, 4), a(5, 4), a(4, 6), a(n - 1, n - 1), a(5, 5)]


def ko_callback(n):
    """``callback`` with the ko fight of ``ko_line`` forced: the prior of black's capture at (4,5) and of white's
    retake at (4,4) is raised to 1000 (before the search renormalises), so descents take, play elsewhere,
    retake and take again -- the same point is captured and played again on one path.  A function of the
    planes (plane 16 = black to move); identity D4 only."""
    take, retake = 4 * n + 5, 4 * n + 4

    def cb(feats, hashes=None):
        pi, v = callback(feats)
        black = feats[:, 16, 0, 0] == 1
        pi[black, take] = 1000.0
        pi[~black, retake] = 1000.0
        return pi, v
    return cb


def prepare(gb, refs, lines=None, handicap=None):
    """play ``lines`` (equal lengths) on the batch and the reference states (RefStateProxy), or place
    ``handicap`` stone lists"""
    if handicap is not None:
        assert all(o.all() for o in gb.place_handicap(handicap))
        for r, s in zip(refs, handicap):
            assert all(r.w("place_handicap", r.k, int(a)) for a in s)
        return
    for t in range(len(lines[0])):
        acts = np.array([ln[t] for ln in lines], np.int32)
        assert gb.forward(acts).all()
        for r, a in zip(refs, acts):
            assert r.forward(int(a))


def run_df_search(gb, mc, n, opts, moves, lines=None, handicap=None, seeds=None, policy_only=False, plane_check=False,
                  net=None, net_name="plain"):
    with RefWorker() as w:
        return _run_df_search(w, gb, mc, n, opts, moves, lines, handicap, seeds, policy_only, plane_check, net, net_name)


def _run_df_search(w, gb, mc, n, opts, moves, lines, handicap, seeds, policy_only, plane_check, net, net_name):
    """``moves`` searched moves of every game of ``gb`` by ``mc`` (a search whose leaf batch is the DF planes)
    and by RefMctsDf on reference states, with a persistent tree: root visit tables, priors (exactly), eval
    counts and the chosen moves must be equal; the reference's move is played.  ``seeds``: reference D4
    streams (``mc`` must run with rotation_flip=1 and a RefStream attached), else rotation_flip=0.
    ``policy_only``: every move is MCTSAI_T::actPolicyOnly's (one wave, the root only).  ``plane_check``: our
    leaves are matched to the reference's evaluated leaves by position hash and the 25 planes compared bit
    for bit.  ``net_name``: the numpy network of both sides (a key of ``NETS``); ``net``: our network instead
    of that one on a host copy of the planes (a torch twin on the device).  The reference runs in a RefWorker.
    Returns the number of leaves whose planes were compared."""
    import torch

    G = gb.num_games
    net_np = NETS[net_name](n)
    refs = [w.state(n) for _ in range(G)]
    prepare(gb, refs, lines, handicap)
    recorded = {}
    flip = 1 if seeds is not None else 0
    rms = [w.search(n, net_name, plane_check, rotation_flip=flip,
                    seed=w("call", "actor_seed", (n, int(seeds[g]))) if flip else 7, **opts) for g in range(G)]
    checked = [0]

    def actor(batch):
        s = batch["s"]
        assert s.dtype == torch.float32 and tuple(s.shape[1:]) == (PLANES, n, n), tuple(s.shape)
        if plane_check:
            h, _, _ = mc.leaf_info()
            x = s.cpu().numpy()
            for i, hh in enumerate(h):
                cands = recorded.get(int(hh))
                assert cands and any((x[i].view(np.uint32) == c.view(np.uint32)).all() for c in cands), \
                    f"leaf planes differ for hash {int(hh):x}"
                checked[0] += 1
        if net is not None:
            return net(batch)
        pi, v = net_np(s.cpu().numpy())
        return {"pi": torch.from_numpy(pi).to(s.device), "V": torch.from_numpy(v).to(s.device)}

    for mv in range(moves):
        want = [rm.act(r, policy_only=policy_only) for rm, r in zip(rms, refs)]
        if plane_check:
            for h, fs in w("recorded").items():
                recorded.setdefault(h, []).extend(fs)
        mc.search(actor, waves=1 if policy_only else None)
        res = mc.results()
        pri = mc.root_priors()
        for g in range(G):
            tag = f"move {mv} game {g}"
            np.testing.assert_array_equal(res["visits"][g], want[g]["visits"], err_msg=f"visits {tag}")
            wp = np.where(want[g]["visits"] >= 0, want[g]["prior"], -1.0).astype(np.float32)
            np.testing.assert_array_equal(pri[g], wp, err_msg=f"priors {tag}")
            assert res["best_action"][g] == want[g]["best_action"], tag
        assert mc.eval_count() == sum(rm.num_evals() for rm in rms), f"eval counts move {mv}"
        acts = np.array([w_["best_action"] for w_ in want], np.int32)
        for r, a in zip(refs, acts):
            assert r.forward(int(a))
        assert gb.forward(acts).all()
        mc.advance(acts)
    return checked[0]
