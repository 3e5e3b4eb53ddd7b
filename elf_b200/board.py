"""GoBatch: a batch of Go games in GPU memory, mirroring the reference ``GoState`` interface.

Reference: ``src_cpp/elfgames/go/base/go_state.h:95-228`` (GoState), ``board.h:289-458`` (Board C
API), ``board_feature.h:61-182`` (BoardFeature).  Each method is the batched counterpart of the
GoState method of the same name and returns one entry per game.
"""
import ctypes

import numpy as np

from . import lib as _l


class GoBatch:
    def __init__(self, num_games, board_size=19, device=0):
        self._lib = _l.load_library()
        self._ctx = _l.vp()
        _l.check(self._lib, self._lib.elfb200_create(board_size, num_games, device, ctypes.byref(self._ctx)))
        self.num_games = num_games
        self.board_size = board_size
        self.num_actions = board_size * board_size + 1
        self.device = device
        self._children = []  # weakrefs to objects holding handles into this context (MctsBatch)

    def new_like(self, num_games):
        """a new batch of ``num_games`` empty games of this batch's board size, on its device and library"""
        gb = GoBatch.__new__(GoBatch)
        gb._lib = self._lib
        gb._ctx = _l.vp()
        _l.check(gb._lib, gb._lib.elfb200_create(self.board_size, num_games, self.device, ctypes.byref(gb._ctx)))
        gb.num_games, gb.board_size, gb.num_actions, gb.device = num_games, self.board_size, self.num_actions, self.device
        gb._children = []
        return gb

    def close(self):
        if getattr(self, "_ctx", None):
            for w in getattr(self, "_children", []):
                c = w()
                if c is not None:
                    c.close()  # search handles reference the context: destroy them first
            self._children = []
            self._lib.elfb200_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- GoState::reset ---------------------------------------------------------------------
    def reset(self, mask=None):
        m = None
        if mask is not None:
            m = np.ascontiguousarray(mask, dtype=np.uint8)
            assert m.shape == (self.num_games,)
        _l.check(self._lib, self._lib.elfb200_reset(self._ctx, m.ctypes.data if m is not None else None))

    # -- GoState::forward -------------------------------------------------------------------
    def forward(self, actions):
        """actions: int array [G]; action = x*N+y, N*N = pass, <0 = leave the game untouched.
        Returns bool array [G]: move accepted (GoState::forward's return value)."""
        a = np.ascontiguousarray(actions, dtype=np.int32)
        assert a.shape == (self.num_games,)
        ok = getattr(self, "_ok_buf", None)
        if ok is None:  # one result buffer per batch (its address is looked up once: this call is latency-critical)
            ok = self._ok_buf = np.empty(self.num_games, np.uint8)
            self._ok_ptr = ok.ctypes.data
        rc = self._lib.elfb200_step(self._ctx, a.__array_interface__["data"][0], self._ok_ptr)
        if rc:
            _l.check(self._lib, rc)
        return ok.view(np.bool_).copy()

    def forward_dev(self, actions_ptr, ok_ptr=None):
        _l.check(self._lib, self._lib.elfb200_step_dev(self._ctx, actions_ptr, ok_ptr))

    def replay(self, move_lists):
        """reset every game and forward its own move list in one launch
        (GoStateExtOffline::switchBeforeMove for the batch); ``move_lists``: G sequences of actions"""
        assert len(move_lists) == self.num_games
        stride = max(1, max((len(m) for m in move_lists), default=1))
        mv = np.full((self.num_games, stride), -1, np.int16)
        cnt = np.zeros(self.num_games, np.int32)
        for g, m in enumerate(move_lists):
            cnt[g] = len(m)
            mv[g, : len(m)] = m
        _l.check(self._lib, self._lib.elfb200_replay(self._ctx, mv.ctypes.data, stride, cnt.ctypes.data))

    def place_handicap(self, stone_lists):
        """GoState::applyHandicap for the batch in one launch: game g places the BLACK stones
        ``stone_lists[g]`` (actions x*N+y) in order, each as PlaceHandicap does.  Only a game still at ply 1
        takes stones; the ply stays 1 and white is to move once a stone is on the board.  Returns one bool
        array per game: PlaceHandicap's verdict for each stone."""
        assert len(stone_lists) == self.num_games
        stride = max(1, max((len(s) for s in stone_lists), default=1))
        st = np.zeros((self.num_games, stride), np.int16)
        cnt = np.zeros(self.num_games, np.int32)
        for g, s in enumerate(stone_lists):
            cnt[g] = len(s)
            st[g, : len(s)] = s
        ok = np.zeros((self.num_games, stride), np.uint8)
        _l.check(self._lib, self._lib.elfb200_place_handicap(self._ctx, st.ctypes.data, stride, cnt.ctypes.data,
                                                             ok.ctypes.data))
        return [ok[g, : cnt[g]].astype(bool) for g in range(self.num_games)]

    # -- GoState's copy constructor -----------------------------------------------------------
    def gather(self, src, index):
        """copy games from the batch ``src`` (same board size and device, not this batch): game i becomes a
        copy of src's game ``index[i]`` for ``index[i]`` in [0, src.num_games); any other value leaves game
        i as it is.  ``index``: G entries, a list / numpy array (synchronous), or an int32 CUDA tensor on
        this batch's device (asynchronous: ordered after the caller's current stream and before its next
        work, with events only, so it can be captured in a CUDA graph).  A search handle on this batch keeps
        its trees: reset the copied games' trees before their next search."""
        if getattr(index, "is_cuda", False):
            return self._gather_dev(src, index)
        a = np.asarray(index)
        if a.dtype != np.int32:  # out-of-range values stay out of range (untouched games) in int32
            a = np.clip(a, -1, src.num_games)
        a = np.ascontiguousarray(a, dtype=np.int32)
        assert a.shape == (self.num_games,)
        _l.check(self._lib, self._lib.elfb200_gather_games(self._ctx, src._ctx, a.ctypes.data))

    def _gather_dev(self, src, index):
        import torch

        dev = torch.device("cuda", self.device)
        if index.dtype != torch.int32 or tuple(index.shape) != (self.num_games,) or not index.is_contiguous() \
                or index.device != dev:
            raise ValueError(f"index must be a contiguous int32 tensor of shape ({self.num_games},) on {dev}")
        if getattr(self, "_gather_ev", None) is None:
            self._gather_ev = [torch.cuda.Event() for _ in range(3)]
            self._gather_stream = torch.cuda.ExternalStream(self.stream, device=dev)
        ev, s_dst = self._gather_ev, self._gather_stream
        s_src = torch.cuda.ExternalStream(src.stream, device=dev)
        cur = torch.cuda.current_stream(dev)
        # both context streams join the caller's stream before the copy and rejoin it afterwards
        ev[0].record(cur)
        s_dst.wait_event(ev[0])
        s_src.wait_event(ev[0])
        _l.check(self._lib, self._lib.elfb200_gather_games_dev(self._ctx, src._ctx, index.data_ptr()))
        ev[1].record(s_dst)
        cur.wait_event(ev[1])
        ev[2].record(s_src)
        cur.wait_event(ev[2])

    def synchronize(self):
        _l.check(self._lib, self._lib.elfb200_synchronize(self._ctx))

    @property
    def stream(self):
        return self._lib.elfb200_stream(self._ctx)

    # -- observers ---------------------------------------------------------------------------
    def getHashCode(self):
        h = np.empty(self.num_games, np.uint64)
        _l.check(self._lib, self._lib.elfb200_get_hash(self._ctx, h.ctypes.data))
        return h

    def info(self):
        """int32 [G,12]: ply, next_player, b_cap, w_cap, last_move, last_move2, ko_action,
        ko_color, 0, terminated, two_pass, superko."""
        o = np.empty((self.num_games, _l.INFO_FIELDS), np.int32)
        _l.check(self._lib, self._lib.elfb200_get_info(self._ctx, o.ctypes.data))
        return o

    def getPly(self):
        return self.info()[:, 0]

    def nextPlayer(self):
        return self.info()[:, 1]

    def terminated(self):
        return self.info()[:, 9].astype(bool)

    def showBoard(self, game=0):
        """GoState::showBoard (go_state.h:187-192) of one game: the reference's board picture"""
        from .online import show_board

        i = self.info()[game]
        return show_board(self.stones()[game], self.board_size, int(i[4]), int(i[2]), int(i[3]), int(i[1]))

    def stones(self):
        n = self.board_size
        o = np.empty((self.num_games, n * n), np.uint8)
        _l.check(self._lib, self._lib.elfb200_get_stones(self._ctx, o.ctypes.data))
        return o

    def legal_mask(self):
        """uint8 [G, N*N+1]: GoState::checkMove for every action (pass always 1)."""
        o = np.empty((self.num_games, self.num_actions), np.uint8)
        _l.check(self._lib, self._lib.elfb200_get_legal(self._ctx, o.ctypes.data))
        return o

    def true_eyes(self, player=0):
        n = self.board_size
        o = np.empty((self.num_games, n * n), np.uint8)
        _l.check(self._lib, self._lib.elfb200_get_true_eyes(self._ctx, player, o.ctypes.data))
        return o

    def tt_score(self):
        o = np.empty(self.num_games, np.int32)
        _l.check(self._lib, self._lib.elfb200_get_tt_score(self._ctx, o.ctypes.data))
        return o

    def evaluate(self, komi=7.5):
        o = np.empty(self.num_games, np.float32)
        _l.check(self._lib, self._lib.elfb200_evaluate(self._ctx, komi, o.ctypes.data))
        return o

    # -- BoardFeature::extractAGZ -----------------------------------------------------------
    def features(self, d4=None):
        n = self.board_size
        o = np.empty((self.num_games, 18, n, n), np.float32)
        d = None
        if d4 is not None:
            d = np.ascontiguousarray(d4, dtype=np.int32)
            assert d.shape == (self.num_games,)
        _l.check(self._lib, self._lib.elfb200_features(self._ctx, d.ctypes.data if d is not None else None, o.ctypes.data))
        return o

    def features_df(self, d4=None):
        """BoardFeature::extract: the 25 DarkForest planes (GameOptions::use_df_feature), float32 [G,25,N,N]"""
        n = self.board_size
        o = np.empty((self.num_games, 25, n, n), np.float32)
        d = None
        if d4 is not None:
            d = np.ascontiguousarray(d4, dtype=np.int32)
            assert d.shape == (self.num_games,)
        _l.check(self._lib, self._lib.elfb200_features_df(self._ctx, d.ctypes.data if d is not None else None, o.ctypes.data))
        return o

    def features_dev(self, out_ptr, d4_ptr=None, fmt=_l.FEAT_F32_NCHW, cpad=0):
        """planes of every game straight into device memory at ``out_ptr``: float32 ``[G,18,N,N]``
        or, in the 16-bit channels-last formats (``lib.FEAT_F16_NHWC`` / ``FEAT_BF16_NHWC``),
        ``[G,N,N,cpad]``.  Asynchronous on the context stream."""
        _l.check(self._lib, self._lib.elfb200_features_dev_ex(self._ctx, d4_ptr, out_ptr, fmt, cpad))

    def set_playout_layout(self, layout):
        """0 = one board row per lane (default), 1 = two rows per lane (19x19: three games per warp)"""
        _l.check(self._lib, self._lib.elfb200_set_playout_layout(self._ctx, int(layout)))

    def set_feature_store(self, mode):
        """16-bit NHWC planes: 0 = direct coalesced 16-byte stores (default), 1 = staged tile + one bulk (TMA) store"""
        _l.check(self._lib, self._lib.elfb200_set_feature_store(self._ctx, int(mode)))

    # -- random-policy playouts (BASELINE configs 1/2/5) ------------------------------------
    def playout(self, seed, first_game_id=0, max_plies=None):
        n = self.board_size
        max_plies = max_plies or 2 * n * n
        G = self.num_games
        chk = np.empty(G, np.uint64)
        plies = np.empty(G, np.int32)
        score = np.empty(G, np.int32)
        fh = np.empty(G, np.uint64)
        tot = ctypes.c_int64()
        _l.check(self._lib, self._lib.elfb200_playout(
            self._ctx, seed, first_game_id, max_plies, chk.ctypes.data, plies.ctypes.data,
            score.ctypes.data, fh.ctypes.data, ctypes.byref(tot)))
        return {"chk": chk, "plies": plies, "score": score, "hash": fh, "total_plies": tot.value}

    def playout_launch(self, seed, first_game_id=0, max_plies=None):
        n = self.board_size
        _l.check(self._lib, self._lib.elfb200_playout_launch(self._ctx, seed, first_game_id, max_plies or 2 * n * n))

    def playout_results(self):
        G = self.num_games
        chk = np.empty(G, np.uint64)
        plies = np.empty(G, np.int32)
        score = np.empty(G, np.int32)
        fh = np.empty(G, np.uint64)
        tot = ctypes.c_int64()
        _l.check(self._lib, self._lib.elfb200_playout_results(
            self._ctx, chk.ctypes.data, plies.ctypes.data, score.ctypes.data, fh.ctypes.data, ctypes.byref(tot)))
        return {"chk": chk, "plies": plies, "score": score, "hash": fh, "total_plies": tot.value}

    def playout_stream(self, seed, first_game_id=0, plies_per_slot=512):
        """steady-state playouts: every slot plays exactly ``plies_per_slot`` plies, restarting
        games as they end; returns per-slot checksum fold / plies / games started / last hash"""
        G = self.num_games
        chk = np.empty(G, np.uint64)
        plies = np.empty(G, np.int32)
        games = np.empty(G, np.int32)
        fh = np.empty(G, np.uint64)
        tot = ctypes.c_int64()
        _l.check(self._lib, self._lib.elfb200_playout_stream(
            self._ctx, seed, first_game_id, plies_per_slot, chk.ctypes.data, plies.ctypes.data,
            games.ctypes.data, fh.ctypes.data, ctypes.byref(tot)))
        return {"chk": chk, "plies": plies, "games": games, "hash": fh, "total_plies": tot.value}

    def playout_stream_launch(self, seed, first_game_id=0, plies_per_slot=512):
        _l.check(self._lib, self._lib.elfb200_playout_stream_launch(self._ctx, seed, first_game_id, plies_per_slot))

    # -- ownership and dead stones -------------------------------------------------------------
    def ownership(self, playouts, seed=0, max_plies=None, out=None, trace=False):
        """Monte-Carlo ownership: ``playouts`` (K) random playouts (the policy of
        include/elfb200_playout_policy.h, draw id g*K + k) from every stored position, which stays as it is.
        Returns int32 ``[G, 2, N*N]`` by action x*N+y: how many playouts end with the point in black's [0] /
        white's [1] area (simple_tt_scoring's view).  A game that ended by two passes is played on; one that
        ended by superko or the ply cap is counted as it stands.  ``trace=True`` also returns the final hash
        (uint64) and plies (int32) of every playout, ``[G, K]`` each.  With ``out``, a contiguous int32 CUDA
        tensor of shape ``[G, 2, N*N]`` on this batch's device, the counts are written there asynchronously,
        ordered after the caller's current stream and before its next work with events only (capturable in a
        CUDA graph after one call of either form has set up the scratch); ``out`` is returned."""
        n, G, K = self.board_size, self.num_games, int(playouts)
        max_plies = 2 * n * n if max_plies is None else int(max_plies)
        seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        if out is not None:
            return self._ownership_dev(K, seed, max_plies, out)
        counts = np.empty((G, 2, n * n), np.int32)
        fh = np.empty((G, K), np.uint64) if trace else None
        pl = np.empty((G, K), np.int32) if trace else None
        _l.check(self._lib, self._lib.elfb200_ownership(
            self._ctx, K, seed, max_plies, counts.ctypes.data, fh.ctypes.data if trace else None,
            pl.ctypes.data if trace else None))
        return (counts, fh, pl) if trace else counts

    def _ownership_dev(self, K, seed, max_plies, out):
        import torch

        dev = torch.device("cuda", self.device)
        n = self.board_size
        if out.dtype != torch.int32 or tuple(out.shape) != (self.num_games, 2, n * n) or not out.is_contiguous() \
                or out.device != dev:
            raise ValueError(f"out must be a contiguous int32 tensor of shape ({self.num_games}, 2, {n * n}) on {dev}")
        if getattr(self, "_own_ev", None) is None:
            self._own_ev = [torch.cuda.Event() for _ in range(2)]
            self._own_stream = torch.cuda.ExternalStream(self.stream, device=dev)
        ev, s = self._own_ev, self._own_stream
        cur = torch.cuda.current_stream(dev)
        ev[0].record(cur)
        s.wait_event(ev[0])
        _l.check(self._lib, self._lib.elfb200_ownership_dev(self._ctx, K, seed, max_plies, out.data_ptr()))
        ev[1].record(s)
        cur.wait_event(ev[1])
        return out

    def final_status(self, counts=None, playouts=None, threshold=0.5):
        """dead groups and getTrompTaylorScore of every stored position.  With ``counts`` (``ownership``'s
        result over ``playouts`` playouts) a group is dead when its stones' mean ownership margin for its own
        colour, (own - opponent) / playouts, is below ``-threshold``; without counts no group is dead.  Returns
        ``(dead, territory, score)``: uint8 ``[G, N*N]`` 1 on dead stones, uint8 ``[G, N*N]`` 1 black / 2 white /
        3 dame with dead stones counted for the opponent, int32 ``[G]`` black minus white (no komi)."""
        n, G = self.board_size, self.num_games
        c = None
        K = 0
        if counts is not None:
            if playouts is None:
                raise ValueError("playouts is required with counts")
            c = np.ascontiguousarray(counts, dtype=np.int32)
            assert c.shape == (G, 2, n * n)
            K = int(playouts)
        dead = np.empty((G, n * n), np.uint8)
        terr = np.empty((G, n * n), np.uint8)
        score = np.empty(G, np.int32)
        _l.check(self._lib, self._lib.elfb200_final_status(
            self._ctx, c.ctypes.data if c is not None else None, K, float(threshold), dead.ctypes.data,
            terr.ctypes.data, score.ctypes.data))
        return dead, terr, score

    def launch_count(self):
        return self._lib.elfb200_launch_count(self._ctx)
