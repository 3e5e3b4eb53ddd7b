"""MctsBatch: the batched GPU tree search, mirroring the reference's MCTSGoAI for G games at once.

Reference: ``src_cpp/elf/ai/tree_search/mcts.h:29-170`` (MCTSAI_T::act), ``tree_search.h``
(TreeSearchT::run / batch_rollouts), ``src_cpp/elfgames/go/mcts/mcts.h:351-381`` (MCTSGoAI) and
the Python NN callback ``src_py/rlpytorch/trainer/trainer.py:73-115`` (Evaluator.actor), whose
contract is kept: ``actor(batch) -> {"pi": [n, N*N+1], "V": [n]}`` with ``batch["s"]`` a CUDA
float tensor ``[n, 18, N, N]``.
"""
import ctypes

import numpy as np

from . import lib as _l
from .refstream import RefStreamSearch

# planes of each leaf-batch format: the 18 AGZ planes, or the 25 DarkForest planes ("df")
_PLANES = {"f32": 18, "f16": 18, "bf16": 18, "df": 25}


class MctsBatch(RefStreamSearch):
    """``feature_format``: "f32" = the GoFeature contract, ``batch["s"]`` float32 ``[n,18,N,N]``
    (default); "f16" / "bf16" = the fast mode for a half-precision channels-last network: the leaf
    batch is written as ``batch["s_nhwc"]`` ``[n,N,N,cpad]`` (planes in channels 0..17, zeros above),
    which ``elf_b200.model.FusedActor`` consumes without a cast/permute pass; "df" = the DarkForest planes
    of ``GameOptions::use_df_feature``, ``batch["s"]`` float32 ``[n,25,N,N]`` (``BoardFeature::extract``).
    ``std_sort_ties=1`` (a search option like the others, ``include/elfb200_mcts.h``): moves whose network
    probabilities are bit-equal are stored in the order ``std::sort`` leaves them in inside the reference's
    ``pi2response`` instead of by ascending move -- needed to replay the reference's games exactly with a
    half-precision network.
    ``strict_root``: raise when a persistent root does not match the board it is asked to search
    (the reference throws, tree_search.h:488-492); off = count it in ``errors()[0]`` and carry on
    with the tree rebuilt from the board."""

    def __init__(self, go_batch, feature_format="f32", cpad=24, strict_root=True, **opts):
        import torch

        self.gb = go_batch
        self._lib = _l.load_library()
        if feature_format not in _PLANES:
            raise ValueError("feature_format must be f32, f16, bf16 or df")
        self.feature_format, self.cpad, self.strict_root = feature_format, int(cpad), bool(strict_root)
        self._mismatches = 0
        o = _l.MctsOptions()
        _l.check(self._lib, self._lib.elfb200_mcts_default_options(ctypes.byref(o)))
        for k, v in opts.items():
            if not hasattr(o, k):
                raise TypeError(f"unknown MCTS option {k}")
            setattr(o, k, v)
        self.options = o
        self._m = _l.vp()
        _l.check(self._lib, self._lib.elfb200_mcts_create(go_batch._ctx, ctypes.byref(o), ctypes.byref(self._m)))
        import weakref

        go_batch._children.append(weakref.ref(self))
        n = go_batch.board_size
        self.waves_per_move = self._lib.elfb200_mcts_waves_per_move(self._m)
        self.max_leaves = self._lib.elfb200_mcts_max_leaves(self._m)
        self._torch = torch
        self.device = torch.device("cuda", go_batch.device)
        # the leaf feature batch handed to the network: lives on the device, written in place
        self.set_feature_format(feature_format, cpad)
        self._stream = torch.cuda.ExternalStream(go_batch.stream, device=self.device)
        self._keep = None  # network replies still being read by kernels on the context stream

    def set_feature_format(self, feature_format, cpad=None):
        """switch the leaf-batch format between moves/waves (re-allocates the feature tensor)"""
        torch = self._torch
        if feature_format not in _PLANES:
            raise ValueError("feature_format must be f32, f16, bf16 or df")
        self.gb.synchronize()
        self.feature_format = feature_format
        self.cpad = self.cpad if cpad is None else int(cpad)
        n = self.gb.board_size
        self.feat = None
        if feature_format in ("f32", "df"):
            self._fmt = _l.FEAT_F32_NCHW if feature_format == "f32" else _l.FEAT_DF_F32_NCHW
            self.feat = torch.zeros((self.max_leaves, _PLANES[feature_format], n, n), dtype=torch.float32,
                                    device=self.device)
        else:
            self._fmt = _l.FEAT_F16_NHWC if feature_format == "f16" else _l.FEAT_BF16_NHWC
            dt = torch.float16 if feature_format == "f16" else torch.bfloat16
            self.feat = torch.zeros((self.max_leaves, n, n, self.cpad), dtype=dt, device=self.device)
        self.feat_key = "s_nhwc" if feature_format in ("f16", "bf16") else "s"

    def close(self):
        if getattr(self, "_m", None):
            # the search handle points into the board context: if that is already gone (interpreter
            # shutdown can finalise objects in any order) the handle must not be touched any more
            if getattr(self.gb, "_ctx", None):
                self._lib.elfb200_mcts_destroy(self._m)
            self._m = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self, mask=None):
        self._ref_settle()
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        _l.check(self._lib, self._lib.elfb200_mcts_reset(self._m, m.ctypes.data if m is not None else None))

    def begin_move(self, active=None):
        self._ref_settle()
        a = None if active is None else np.ascontiguousarray(active, dtype=np.uint8)
        _l.check(self._lib, self._lib.elfb200_mcts_begin_move(self._m, a.ctypes.data if a is not None else None))
        self._ref_begin(a)
        if self.strict_root:
            bad = int(self.errors()[0])
            if bad != self._mismatches:
                n, self._mismatches = bad - self._mismatches, bad
                raise _l.ElfB200Error(
                    f"TreeSearch::Root state is not the same as the input state in {n} game(s): the board moved "
                    "without advance()/reset() of the search (the stale trees were discarded)")

    def select(self, wait=True):
        """one wave of descents; returns the CUDA feature tensor view of the leaves that need the
        network (``[n,18,N,N]`` float32, ``[n,25,N,N]`` with "df", or ``[n,N,N,cpad]`` in the 16-bit
        formats; n may be 0).
        ``wait=False``: nothing is read back and the host does not wait -- the view covers all
        ``max_leaves`` rows (rows past the device-side count are stale, their replies are ignored);
        ``leaf_count()`` fetches the count later."""
        n = ctypes.c_int32()
        _l.check(self._lib, self._lib.elfb200_mcts_select_ex(self._m, self.feat.data_ptr(), self._fmt, self.cpad,
                                                             ctypes.byref(n) if wait else None))
        self._n = n.value if wait else -1
        return self.feat[: n.value] if wait else self.feat

    def leaf_features_again(self, out=None, fmt=None, cpad=None):
        """write the planes of the pending leaves once more (default: into the batch tensor, same
        format); asynchronous on the context stream"""
        t = self.feat if out is None else out
        _l.check(self._lib, self._lib.elfb200_mcts_leaf_features(self._m, t.data_ptr(), self._fmt if fmt is None else fmt,
                                                                 self.cpad if cpad is None else cpad))

    def leaf_count(self):
        n = ctypes.c_int32()
        _l.check(self._lib, self._lib.elfb200_mcts_leaf_count(self._m, ctypes.byref(n)))
        return n.value

    def leaf_info(self):
        n = self._n
        h = np.empty(n, np.uint64)
        g = np.empty(n, np.int32)
        p = np.empty(n, np.int32)
        self.leaf_d4 = np.empty(n, np.int32)
        _l.check(self._lib, self._lib.elfb200_mcts_leaf_info(self._m, h.ctypes.data, g.ctypes.data, p.ctypes.data,
                                                             self.leaf_d4.ctypes.data))
        return h, g, p

    def expand_backup(self, pi, v):
        """pi: CUDA float32 [n, N*N+1], v: CUDA float32 [n] (contiguous), produced on any stream
        the caller has synchronised with the context stream."""
        if self._n != 0:
            assert pi.is_cuda and v.is_cuda and pi.dtype == self._torch.float32 and v.dtype == self._torch.float32
            assert pi.is_contiguous() and v.is_contiguous()
            assert pi.shape[0] >= (self._n if self._n > 0 else self.max_leaves)
            _l.check(self._lib, self._lib.elfb200_mcts_expand_backup(self._m, pi.data_ptr(), v.data_ptr()))
            # the kernels read pi / v on the context stream, which the caching allocator knows nothing
            # about: keep the tensors alive until the next wave has been ordered behind them
            self._keep = (pi, v)
        else:
            _l.check(self._lib, self._lib.elfb200_mcts_expand_backup(self._m, None, None))

    def results(self):
        G, P1 = self.gb.num_games, self.gb.num_actions
        best = np.empty(G, np.int32)
        visits = np.empty((G, P1), np.int32)
        rootv = np.empty(G, np.float32)
        bestq = np.empty(G, np.float32)
        tot = np.empty(G, np.int32)
        _l.check(self._lib, self._lib.elfb200_mcts_results(
            self._m, best.ctypes.data, visits.ctypes.data, rootv.ctypes.data, bestq.ctypes.data, tot.ctypes.data))
        return {"best_action": best, "visits": visits, "root_value": rootv, "best_q": bestq, "total_visits": tot}

    def choose(self, policy_distri_cutoff, resign_thres, never_resign=None, seed=0):
        """device-side move choice (sample ~ visits while ply <= cutoff, else most visited; -1 =
        resign, -2 = not searched); returns (actions int32[G], values float32[G])"""
        G = self.gb.num_games
        a = np.empty(G, np.int32)
        v = np.empty(G, np.float32)
        nr = None if never_resign is None else np.ascontiguousarray(never_resign, dtype=np.uint8)
        _l.check(self._lib, self._lib.elfb200_mcts_choose(
            self._m, int(policy_distri_cutoff), float(resign_thres), nr.ctypes.data if nr is not None else None,
            int(seed) & 0xFFFFFFFFFFFFFFFF, a.ctypes.data, v.ctypes.data))
        return a, v

    def advance(self, actions):
        self._ref_settle()
        a = np.ascontiguousarray(actions, dtype=np.int32)
        _l.check(self._lib, self._lib.elfb200_mcts_advance(self._m, a.ctypes.data))

    # -- copying trees between handles -----------------------------------------------------------
    def gather(self, src, index):
        """copy search trees from the handle ``src`` (same board size and ``nodes_per_game``, not this handle;
        it may search the same GoBatch): game i's tree becomes an exact replica of src's game ``index[i]`` for
        ``index[i]`` in [0, src's number of games); any other value leaves game i's tree as it is.  Continued
        search on a copy is bitwise the search its source would run.  The random state of each game (D4 codes,
        root noise) stays with this handle.  ``index`` as in ``GoBatch.gather``: a list / numpy array
        (synchronous) or a contiguous int32 CUDA tensor on this handle's device (asynchronous: ordered after the
        caller's current stream and before its next work, with events only, so it can be captured in a CUDA
        graph).  Not while either handle has a wave open (``select`` without ``expand_backup``).

        Copy the boards with the same index first (``GoBatch.gather`` / ``GoEnv.load``): the next
        ``begin_move`` checks every root against its board, so a tree whose board was not copied raises with
        ``strict_root`` or is counted in ``errors()[0]`` and rebuilt from the board."""
        if getattr(index, "is_cuda", False):
            return self._gather_dev(src, index)
        G = self.gb.num_games
        a = np.asarray(index)
        if a.dtype != np.int32:  # out-of-range values stay out of range (untouched games) in int32
            a = np.clip(a, -1, src.gb.num_games)
        a = np.ascontiguousarray(a, dtype=np.int32)
        if a.shape != (G,):
            raise ValueError(f"index must have shape ({G},), got {a.shape}")
        _l.check(self._lib, self._lib.elfb200_mcts_gather(self._m, src._m, a.ctypes.data))

    def _gather_dev(self, src, index):
        torch = self._torch
        G = self.gb.num_games
        if index.dtype != torch.int32 or tuple(index.shape) != (G,) or not index.is_contiguous() \
                or index.device != self.device:
            raise ValueError(f"index must be a contiguous int32 tensor of shape ({G},) on {self.device}")
        if getattr(self, "_gather_ev", None) is None:
            self._gather_ev = [torch.cuda.Event() for _ in range(3)]
        ev, s_dst, s_src = self._gather_ev, self._stream, src._stream
        cur = torch.cuda.current_stream(self.device)
        # both context streams join the caller's stream before the copy and rejoin it afterwards
        ev[0].record(cur)
        s_dst.wait_event(ev[0])
        s_src.wait_event(ev[0])
        _l.check(self._lib, self._lib.elfb200_mcts_gather_dev(self._m, src._m, index.data_ptr()))
        ev[1].record(s_dst)
        cur.wait_event(ev[1])
        ev[2].record(s_src)
        cur.wait_event(ev[2])

    # -- search without the host: the device forms (elfb200_mcts_*_dev) -----------------------------------------
    def _check_dev(self, t, dtypes, shape, name):
        if t.device != self.device or t.dtype not in dtypes or tuple(t.shape) != shape or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous {'/'.join(map(str, dtypes))} tensor of shape {shape} on "
                             f"{self.device}")

    def _mask_dev(self, mask, name):
        if mask is None:
            return None
        torch = self._torch
        self._check_dev(mask, (torch.uint8, torch.bool), (self.gb.num_games,), name)
        return mask.view(torch.uint8).data_ptr()

    def _dev_call(self, call):
        """``call`` on the context stream, ordered after the caller's current stream and before its next work:
        events only, no host synchronisation (as ``GoEnv`` orders its calls)"""
        cuda = self.device.type == "cuda"
        if cuda:
            if getattr(self, "_dev_ev", None) is None:
                self._dev_ev = [self._torch.cuda.Event(), self._torch.cuda.Event()]
            cur = self._torch.cuda.current_stream(self.device)
            self._dev_ev[0].record(cur)
            self._stream.wait_event(self._dev_ev[0])
        call()
        if cuda:
            self._dev_ev[1].record(self._stream)
            cur.wait_event(self._dev_ev[1])

    def _dev_out(self):
        """the fixed output tensors of choose_dev / results_dev, allocated on first use"""
        if getattr(self, "_dev_tables", None) is None:
            torch, G, P1, d = self._torch, self.gb.num_games, self.gb.num_actions, self.device
            i32, f32 = torch.int32, torch.float32
            self._dev_tables = {
                "actions": torch.zeros(G, dtype=i32, device=d), "values": torch.zeros(G, dtype=f32, device=d),
                "best_action": torch.zeros(G, dtype=i32, device=d), "visits": torch.zeros((G, P1), dtype=i32, device=d),
                "root_value": torch.zeros(G, dtype=f32, device=d), "best_q": torch.zeros(G, dtype=f32, device=d),
                "total_visits": torch.zeros(G, dtype=i32, device=d)}
        return self._dev_tables

    def search_dev(self, actor, move, active=None):
        """One whole move (``begin_move`` and ``waves_per_move`` waves) without the host: nothing is read back and
        the host never waits, so the call can be captured in a CUDA graph -- a graph must hold whole moves, because
        each wave's D4 codes are keyed by the wave index, which the host passes by value.

        ``move``: int64 [1] tensor on this handle's device, the move index that keys the root noise (the host form
        keys it by a host counter, which would be frozen in a graph: advance the tensor, e.g. ``move.add_(1)``,
        so that every replay draws fresh noise).  ``active``: uint8 / bool [G] tensor, or None (all games).

        ``actor(batch) -> {"pi", "V"}`` is called every wave on the full ``max_leaves`` feature view
        (``batch[self.feat_key]``); rows past the device-side leaf count are stale and their replies are ignored.
        Inside a capture the actor must itself be capturable: no host synchronisation and no graph of its own.
        ``FusedActor(cuda_graph=True)`` replays its own graph, so it can only be used uncaptured; plain
        ``PolicyValueNet``, ``Actor`` and ``FusedActor(cuda_graph=False)`` should be capturable, which is not
        verified here (``scripts/search_graph_bench.py`` captures the actor it uses).

        Ordering with the caller's current stream uses events only.  There is no ``strict_root`` check: a root
        that does not match its board is counted in ``errors()[0]`` and rebuilt.  Host-side counters do not see
        work replayed from a graph (``timings``); the device counters (``stats``, ``errors``, ``eval_count``) do."""
        torch = self._torch
        self._check_dev(move, (torch.int64,), (1,), "move")
        act = self._mask_dev(active, "active")
        cuda = self.device.type == "cuda"
        L, m = self._lib, self._m
        self._dev_call(lambda: _l.check(L, L.elfb200_mcts_begin_move_dev(m, act, move.data_ptr())))
        for _ in range(self.waves_per_move):
            self._dev_call(lambda: _l.check(L, L.elfb200_mcts_select_dev(m, self.feat.data_ptr(), self._fmt, self.cpad)))
            with torch.no_grad():
                reply = actor({self.feat_key: self.feat})
                pi = reply["pi"].to(torch.float32).contiguous()
                v = reply["V"].to(torch.float32).reshape(-1).contiguous()
            if pi.shape[0] < self.max_leaves or v.shape[0] < self.max_leaves or pi.device != self.device:
                raise ValueError(f"the actor must answer all {self.max_leaves} rows on {self.device}")
            self._dev_call(lambda: _l.check(L, L.elfb200_mcts_expand_backup_dev(m, pi.data_ptr(), v.data_ptr())))
            # the reply is read on the context stream, which the caching allocator knows nothing about
            self._keep = (pi, v) if cuda else None

    def choose_dev(self, policy_distri_cutoff, resign_thres, seed, never_resign=None):
        """``choose`` with the seed read from ``seed`` (int64 [1] tensor on this handle's device) when the kernel
        runs, so a graph replay draws with the seed the tensor then holds; ``never_resign``: uint8 / bool [G]
        tensor or None.  Returns this handle's fixed (actions int32 [G], values float32 [G]) tensors: their
        addresses stay the same across calls, and each call overwrites them."""
        torch = self._torch
        self._check_dev(seed, (torch.int64,), (1,), "seed")
        nr = self._mask_dev(never_resign, "never_resign")
        out = self._dev_out()
        a, v = out["actions"], out["values"]
        L, m = self._lib, self._m
        self._dev_call(lambda: _l.check(L, L.elfb200_mcts_choose_dev(
            m, int(policy_distri_cutoff), float(resign_thres), nr, seed.data_ptr(), a.data_ptr(), v.data_ptr())))
        return a, v

    def results_dev(self):
        """``results`` into this handle's fixed tensors on its device (the same dict of tensors every call)"""
        o = self._dev_out()
        r = {k: o[k] for k in ("best_action", "visits", "root_value", "best_q", "total_visits")}
        L, m = self._lib, self._m
        self._dev_call(lambda: _l.check(L, L.elfb200_mcts_results_dev(
            m, *(r[k].data_ptr() for k in ("best_action", "visits", "root_value", "best_q", "total_visits")))))
        return r

    def advance_dev(self, actions):
        """``advance`` from an int32 [G] tensor on this handle's device (< 0: the game's tree is untouched)"""
        torch = self._torch
        self._check_dev(actions, (torch.int32,), (self.gb.num_games,), "actions")
        L, m = self._lib, self._m
        self._dev_call(lambda: _l.check(L, L.elfb200_mcts_advance_dev(m, actions.data_ptr())))

    def reset_dev(self, mask=None):
        """``reset`` for the games where the uint8 / bool [G] tensor ``mask`` is set (None: every game)"""
        mp = self._mask_dev(mask, "mask")
        L, m = self._lib, self._m
        self._dev_call(lambda: _l.check(L, L.elfb200_mcts_reset_dev(m, mp)))

    def tree_usage(self):
        """(nodes, edges) int32 [G] each: in-use nodes and stored edges of the visited nodes of every game's
        tree, the records ``gather`` copies for the game"""
        G = self.gb.num_games
        nodes, edges = np.zeros(G, np.int32), np.zeros(G, np.int32)
        _l.check(self._lib, self._lib.elfb200_mcts_tree_usage(self._m, nodes.ctypes.data, edges.ctypes.data))
        return nodes, edges

    def root_priors(self):
        """float32 [G, N*N+1]: prior of every root edge by action, -1 where there is no edge"""
        o = np.empty((self.gb.num_games, self.gb.num_actions), np.float32)
        _l.check(self._lib, self._lib.elfb200_mcts_root_priors(self._m, o.ctypes.data))
        return o

    def errors(self):
        e = np.zeros(4, np.int32)
        _l.check(self._lib, self._lib.elfb200_mcts_errors(self._m, e.ctypes.data))
        return e

    def eval_count(self):
        return self._lib.elfb200_mcts_eval_count(self._m)

    def timings(self, reset=False):
        """(ms[4] = select, features, expand, backup kernel time; number of waves)"""
        ms = np.zeros(4, np.float64)
        w = ctypes.c_int64()
        _l.check(self._lib, self._lib.elfb200_mcts_timings(self._m, ms.ctypes.data, ctypes.byref(w), int(reset)))
        return ms, w.value

    def stats(self):
        """uint64[4]: descent steps, edge records read, nodes created, stored edges of visited nodes"""
        s = np.zeros(4, np.uint64)
        _l.check(self._lib, self._lib.elfb200_mcts_stats(self._m, s.ctypes.data))
        return s

    # -- MCTSAI_T::act for all games -----------------------------------------------------------
    def act(self, actor, active=None):
        """Run one full search (all waves) with ``actor(batch) -> {"pi", "V"}`` as the network
        callback and return the root statistics.  The callback sees ``batch["s"]`` on the GPU."""
        self.search(actor, active)
        return self.results()

    def wave(self, actor):
        """one wave: descents, the network on the claimed leaves, expansion and backup.  The host
        waits once (for the leaf count); network and search kernels are ordered by stream events."""
        self.wave_finish(self.wave_eval(actor, self.wave_select()))

    # -- the three pieces of a wave (elf_b200.pipeline.WavePipeline interleaves them across batches) --
    def wave_select(self):
        """descents + leaf features; returns the (padded) feature view for the network or None"""
        pad = int(getattr(self, "_pad", 0) or 0)
        s = self.select()  # waits for the context stream to learn the leaf count
        if s.shape[0] == 0:
            return None
        if pad > 1:
            # static NN shapes: round the batch up to a multiple of the actor's batch size
            # (rows past n are stale features; their replies are never read)
            s = self.feat[: min(-(-s.shape[0] // pad) * pad, self.max_leaves)]
        return s

    def wave_eval(self, actor, s, nn_stream=None):
        """enqueue the network on ``nn_stream`` (default: torch's current stream) behind the feature
        kernel; returns (pi, v, event) or None"""
        if s is None:
            return None
        torch = self._torch
        st = nn_stream if nn_stream is not None else torch.cuda.current_stream(self.device)
        st.wait_stream(self._stream)  # the network after the features
        with torch.cuda.stream(st), torch.no_grad():
            reply = actor({self.feat_key: s})
            pi = reply["pi"].to(torch.float32).contiguous()
            v = reply["V"].to(torch.float32).reshape(-1).contiguous()
            ev = torch.cuda.Event()
            ev.record(st)
        return pi, v, ev

    def wave_finish(self, reply):
        """expansion + backup on the context stream, behind the network's event; does not wait"""
        if reply is None:
            self.expand_backup(None, None)
            return
        pi, v, ev = reply
        self._stream.wait_event(ev)
        self.expand_backup(pi, v)

    def search(self, actor, active=None, waves=None):
        """the search of ``act`` without fetching the root tables (use ``choose`` / ``results``).
        ``waves``: run only that many waves (1 on a fresh tree = evaluate and expand the root only,
        TreeSearchT::runPolicyOnly, tree_search.h:387-408); default: the whole move"""
        self.begin_move(active)
        self._pad = int(getattr(actor, "batchsize", 0) or 0)
        for _ in range(self.waves_per_move if waves is None else int(waves)):
            self.wave(actor)
