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

    def launch_count(self):
        return self._lib.elfb200_launch_count(self._ctx)
