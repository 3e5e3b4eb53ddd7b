"""SelfPlay: the per-move driver of the reference's self-play game loop, for G games at once.

Mirrors ``GoGameSelfPlay::act`` (``src_cpp/elfgames/go/common/game_selfplay.cc:272-430``):
one MCTS per move, ``mcts_make_diverse_move`` (sample from the visit distribution while
``ply <= policy_distri_cutoff``, ``:80-95``), ``MCTSGoAI::getValue`` as predicted value,
``ResignCheck`` (``common/game_utils.h:15-54``: resign when the side to move's value is below
``-1 + resign_thres`` and ``ply >= 50``; a ``never_resign_ratio`` fraction of games never resigns),
``GoState::forward``, game end on two passes / ply cap / superko / ``move_cutoff`` with the final
value from ``GoState::evaluate(komi)`` (``go_state_ext.h:79-105``), then restart.

Randomness: by default move sampling runs on the device (counter-based generator) and the
never-resign draw comes from a numpy Generator -- the reference's distributions, not its streams.
``rng="reference"`` switches to the reference's own streams (``elf_b200.refstream``): every game
owns the two ``std::mt19937`` generators of a reference game thread seeded from ``seed``
(``GameOptions::seed``; an array gives every game its own), root noise / D4 codes / sampled moves /
the never-resign draw consume them exactly where ``GoGameSelfPlay::act`` does, and ties between
equally visited moves resolve in the reference's container order: the batch then plays, move for
move, the games the reference's game threads play with that seed (single search thread).  With a
network whose replies hold bit-equal probabilities (half precision: equal logits) add the search
option ``std_sort_ties=1``, which stores such moves in the order ``std::sort`` leaves them in.
"""
import numpy as np

from .board import GoBatch
from .mcts import MctsBatch


class SelfPlay:
    def __init__(self, actor, num_games=4096, board_size=19, device=0, policy_distri_cutoff=20,
                 resign_thres=0.05, never_resign_ratio=0.1, move_cutoff=-1, komi=7.5, seed=0,
                 record_games=False, actor_white=None, board=None, search=None, search_white=None,
                 white_mcts_opts=None, black_use_policy_network_only=False, white_use_policy_network_only=False,
                 policy_distri_training_for_all=False, num_games_per_thread=-1, rng="numpy", use_df_feature=False,
                 **mcts_opts):
        # board / search / search_white: pre-built GoBatch / MctsBatch objects (or duck-typed stand-ins:
        # the CPU tests of the host logic inject oracle-backed ones); by default they are created here
        # use_df_feature (GameOptions::use_df_feature): both AIs search on the 25 DarkForest planes, "s" float32
        # [n,25,N,N] (a policy-only colour evaluates its root through the same leaf batch)
        self.use_df_feature = bool(use_df_feature)
        if self.use_df_feature:
            for o in (mcts_opts, white_mcts_opts or {}):
                if o.get("feature_format", "df") not in ("f32", "df"):
                    raise ValueError("use_df_feature writes float32 DarkForest planes: feature_format "
                                     f"{o['feature_format']!r} is not available with it")
            mcts_opts["feature_format"] = "df"
            if white_mcts_opts and "feature_format" in white_mcts_opts:
                white_mcts_opts = {**white_mcts_opts, "feature_format": "df"}
        self.gb = board if board is not None else GoBatch(num_games, board_size=board_size, device=device)
        mcts_opts.setdefault("komi", komi)
        self._mcts_opts = dict(mcts_opts)
        # the second AI may search differently (GameOptions::white_puct / white_mcts_rollout_per_batch /
        # white_mcts_rollout_per_thread, game_selfplay.cc:175-182): overrides on top of the common options
        self._white_opts = {**mcts_opts, **(white_mcts_opts or {})}
        if rng not in ("numpy", "reference"):
            raise ValueError("rng must be 'numpy' or 'reference'")
        self.ref = None
        if rng == "reference":
            from .refstream import RefStream

            self.ref = RefStream(num_games, board_size, seed)
            self._ref_started = False  # the actors are seeded at the first restart() (game_selfplay.cc:151-200)
            self._nr_drawn = np.zeros(num_games, bool)  # ResignCheck::has_calculated_never_resign
            seed = int(np.asarray(seed).reshape(-1)[0])
        self.mcts = search if search is not None else self._make_search(mcts_opts, 0)
        if search is not None and self.ref is not None:
            search.attach_ref_stream(self.ref, 0, float(mcts_opts.get("root_epsilon", 0)), float(mcts_opts.get("root_alpha", 0)))
        self.actor = actor
        # evaluation matches (GoGameSelfPlay::_ai2, game_selfplay.cc:366-367): a second AI with its own
        # tree plays white; both trees follow every move (MCTSAI_T::advanceMoves)
        self.actor_white = actor_white
        if search_white is not None:
            self.mcts2 = search_white
            if self.ref is not None:
                search_white.attach_ref_stream(self.ref, 1, float(self._white_opts.get("root_epsilon", 0)),
                                               float(self._white_opts.get("root_alpha", 0)))
        else:
            self.mcts2 = self._make_search(self._white_opts, 1) if (actor_white is not None and search is None) else None
        # server requests (MsgRequest: model versions + client control), see set_request()
        self.request = {"black_ver": -1, "white_ver": -1, "player_swap": False, "async": False,
                        "num_game_thread_used": -1}
        # GameOptions::black/white_use_policy_network_only (game_selfplay.cc:360-371): that colour moves by
        # the network policy alone (MCTSAI_T::actPolicyOnly), no search
        self.policy_only = {1: bool(black_use_policy_network_only), 2: bool(white_use_policy_network_only)}
        self.protocol = False  # becomes True with the first set_request()
        self.idle = None  # bool[G]: games that wait for a request (ModelPair::wait); None = nobody waits
        self.swap = False  # player_swap of an evaluation match: the "white" AI plays black
        self.G = num_games
        self.N = board_size
        self.komi = komi
        self.policy_distri_cutoff = policy_distri_cutoff
        self.resign_thres = resign_thres
        self.never_resign_ratio = never_resign_ratio
        self.move_cutoff = move_cutoff
        self.rng = np.random.default_rng(seed)
        self._seed = int(seed)
        self._move_counter = 0
        self.never_resign = (self.rng.random(num_games) < never_resign_ratio) if self.ref is None else np.zeros(num_games, bool)
        self.moves_played = 0
        self.games_finished = 0
        self.results = []  # (final_value, plies, reason) of finished games
        self.records = []  # reference-format game records (elf_b200.record) when record_games is on
        self.recorders = None
        if record_games:
            from .record import GameRecorder

            self.recorders = [GameRecorder(board_size, g, policy_distri_cutoff, policy_distri_training_for_all,
                                           mcts_opt=self._mcts_opts) for g in range(num_games)]
        # GameOptions::num_games_per_thread (GoStateExt::finished, go_state_ext.h:229-232): a game slot
        # stops after that many games (-1: never); stopped slots idle like parked ones
        self.num_games_per_thread = int(num_games_per_thread)
        self.games_per_slot = np.zeros(num_games, np.int64)
        self.stopped = np.zeros(num_games, bool)

    def _make_search(self, opts, which):
        """the search of AI ``which`` (0 = _ai, 1 = _ai2); under rng='reference' its root noise is drawn
        on the host from that AI's generator, so the device's own noise stays off"""
        if self.ref is None:
            return MctsBatch(self.gb, **opts)
        o = dict(opts)
        eps, alpha = float(o.pop("root_epsilon", 0.0)), float(o.pop("root_alpha", 0.0))
        mc = MctsBatch(self.gb, **o)
        mc.attach_ref_stream(self.ref, which, eps, alpha)
        return mc

    def _ref_start(self):
        """GoGameSelfPlay::restart for a batch that never saw a request: init_ai seeds _ai (and _ai2)
        from the game generator (game_selfplay.cc:47,165-182)"""
        if self.ref is not None and not self._ref_started:
            self.ref.init_actor(0)
            if self.mcts2 is not None:
                self.ref.init_actor(1)
            self._ref_started = True

    def _choose_reference(self, info):
        """mcts_make_diverse_move + mcts_update_info + shouldResign (game_selfplay.cc:80-101,387-391) on
        the reference's streams: returns (actions, values) like ``MctsBatch.choose``"""
        G = self.G
        searched = np.ones(G, bool) if self.idle is None else ~self.idle
        sample = info[:, 0] <= self.policy_distri_cutoff
        if self.mcts2 is None:
            c = self.mcts.ref_choose(sample, mask=searched.astype(np.uint8))
            acts, vals = c["action"].copy(), c["value"].copy()
        else:
            first = (info[:, 1] == 1) != self.swap  # games whose mover was searched by self.mcts (see phases)
            c1 = self.mcts.ref_choose(sample, mask=(searched & first).astype(np.uint8))
            c2 = self.mcts2.ref_choose(sample, mask=(searched & ~first).astype(np.uint8))
            acts = np.where(first, c1["action"], c2["action"]).astype(np.int32)
            vals = np.where(first, c1["value"], c2["value"]).astype(np.float32)
        self._resign_reference(info, acts, vals, searched)
        acts[~searched] = -2
        return acts, vals

    def _resign_reference(self, info, acts, vals, searched):
        """GoStateExt::shouldResign on the reference's streams, in place on ``acts`` (-1 = resign).
        ResignCheck::check: the first call of a game draws never_resign from the game generator
        (game_utils.h:25-30); it is called every move, whatever the ply (game_selfplay.cc:387)"""
        need = searched & ~self._nr_drawn
        if need.any():
            u = self.ref.game_uniform(need.astype(np.uint8))
            self.never_resign[need] = u[need] < float(np.float32(self.never_resign_ratio))
            self._nr_drawn |= need
        self._resign(info, acts, vals, searched)

    def _resign(self, info, acts, vals, sel):
        """ResignCheck::check after the never-resign draw, for the games in ``sel``: resign unless
        ``value >= -1 + resign_thres`` (game_utils.h:36-39, a float compared in double; written the
        reference's way round, so a NaN value -- the 0/0 of an unvisited edge, see policy_only_plan --
        resigns as it does there) and only from ply 50 on (game_selfplay.cc:388)"""
        side = np.where(info[:, 1] == 1, vals, -vals).astype(np.float64)
        resign = sel & ~self.never_resign & ~(side >= -1.0 + float(np.float32(self.resign_thres))) & (info[:, 0] >= 50)
        acts[resign] = -1

    def close(self):
        self.mcts.close()
        if self.mcts2 is not None:
            self.mcts2.close()
        self.gb.close()

    @staticmethod
    def merge_results(black_to_move, res_b, res_w):
        """root statistics of the AI that is to move in each game"""
        out = {}
        for k in res_b:
            m = black_to_move if res_b[k].ndim == 1 else black_to_move[:, None]
            out[k] = np.where(m, res_b[k], res_w[k])
        return out

    def phases(self, info):
        """which AI searches which games this move: [(search, actor, label, active mask or None)].
        One AI for self-play; for a match ``_ai`` (label actor_black) takes the black-to-move games
        and ``_ai2`` (actor_white) the others -- the other way round under player_swap
        (GoGameSelfPlay::restart swaps the two pointers, game_selfplay.cc:185-188)."""
        self._ref_start()
        act = None if self.idle is None else ~self.idle
        if self.mcts2 is None:
            return [(self.mcts, self.actor, "actor_black", None if act is None else act.astype(np.uint8))]
        first = (info[:, 1] == 1) != self.swap  # games whose side to move is served by _ai's model
        second = ~first
        if act is not None:
            first, second = first & act, second & act
        return [(self.mcts, self.actor, "actor_black", first.astype(np.uint8)),
                (self.mcts2, self.actor_white, "actor_white", second.astype(np.uint8))]

    def step(self):
        """one move of every game; returns the number of moves played"""
        info = self.gb.info()
        self._ref_start()
        if self.policy_only[1] or self.policy_only[2]:
            return self.finish_move(info, chosen=self._search_with_policy_only(info))
        if self.mcts2 is None and self.idle is None:
            self.mcts.search(self.actor)
        else:
            for mc, actor, _, active in self.phases(info):
                mc.search(actor, active=active)
        return self.finish_move(info)

    def policy_only_plan(self, info, acts, vals):
        """The search phases of a move in which one colour moves by policy only, as a list of
        ``(search, actor, label, active mask, waves, post)``: run ``waves`` waves (None = a whole
        move's, 0 = none) for the games in ``active``, then call ``post()``, which fills ``acts`` /
        ``vals`` for those games.  Policy-only games get their root evaluated if it is not yet
        (TreeSearchT::runPolicyOnly, tree_search.h:387-408: no root noise, one D4 draw if the network is
        asked) and play the edge with the largest prior (rank criterion PRIOR, first maximum in the
        reference's container order); the other games search as usual.  The predicted value of a
        policy-only move is MCTSGoAI::getValue of that result (go/mcts/mcts.h:358-365): the root's
        network value while the root edges have no visits, else W/N of the CHOSEN edge -- in a tree
        shared with a searching colour the root usually has visits, and an unvisited largest-prior edge
        then yields 0/0 = NaN, which ResignCheck::check treats as "resign" (see ``_resign``).  Callers
        switch the reference-stream root noise off for the phases whose ``waves`` is not None
        (``set_root_noise_enabled``).  Shared by ``step()`` and the wait/step pump of ``compat``."""
        G = self.G
        po_colour = np.array([self.policy_only[int(c)] for c in info[:, 1]], bool)
        nr = self.never_resign.astype(np.uint8)
        seed = (self._seed << 20) ^ (self._move_counter + 1)
        sample = info[:, 0] <= self.policy_distri_cutoff
        plan = []
        for mc, actor, label, active in self.phases(info):
            act = np.ones(G, bool) if active is None else np.asarray(active).astype(bool)
            a_po, a_ts = act & po_colour, act & ~po_colour
            if a_ts.any():
                def post_ts(mc=mc, sel=a_ts):
                    if self.ref is not None:  # the resign check follows in finish_move (_resign_reference)
                        c = mc.ref_choose(sample, mask=sel.astype(np.uint8))
                        a, v = c["action"], c["value"]
                    else:
                        a, v = mc.choose(self.policy_distri_cutoff, self.resign_thres, nr, seed)
                    acts[sel], vals[sel] = a[sel], v[sel]
                plan.append((mc, actor, label, a_ts.astype(np.uint8), None, post_ts))
            if a_po.any():
                # roots that are already expanded (left by the other colour's search in a shared tree)
                # are used as they are; the others are evaluated once
                fresh = a_po & (mc.root_priors().max(1) < 0)

                def post_po(mc=mc, sel=None):
                    e = mc.root_edges()
                    rv = mc.results()["root_value"]
                    for g in np.flatnonzero(sel):
                        n = int(e["n_edges"][g])
                        b = self.first_largest(e["priors"][g, :n], e["actions"][g, :n])
                        acts[g] = int(e["actions"][g, b])
                        if int(e["visits"][g, :n].sum()) == 0:
                            vals[g] = rv[g]
                        else:
                            with np.errstate(divide="ignore", invalid="ignore"):
                                vals[g] = e["wsum"][g, b] / np.float32(e["visits"][g, b])  # EdgeInfo::getQSA
                    if self.ref is None:
                        self._resign(info, acts, vals, sel)
                old = a_po & ~fresh
                if old.any():
                    plan.append((mc, actor, label, old.astype(np.uint8), 0, lambda f=post_po, m=old: f(sel=m)))
                if fresh.any():
                    plan.append((mc, actor, label, fresh.astype(np.uint8), 1, lambda f=post_po, m=fresh: f(sel=m)))
        self._po_colour = po_colour
        return plan

    def first_largest(self, scores, actions):
        """storage index of the edge MCTSResultT::addActions picks (tree_search_base.h:237-294): the first
        strict maximum of ``scores`` walking the edges in the reference's container order"""
        top = np.flatnonzero(scores == scores.max())
        if len(top) == 1:
            return int(top[0])
        from .refstream import RefStream

        is_top = np.zeros(len(scores), bool)
        is_top[top] = True
        for i in RefStream.edge_order(self.N, actions):
            if is_top[i]:
                return int(i)

    def _search_with_policy_only(self, info):
        """the search phase when one colour moves by policy only (see policy_only_plan); returns the
        chosen (actions, values) for finish_move"""
        acts = np.full(self.G, -2, np.int32)
        vals = np.zeros(self.G, np.float32)
        for mc, actor, _, active, waves, post in self.policy_only_plan(info, acts, vals):
            mc.set_root_noise_enabled(waves is None)
            try:
                if waves == 0:
                    mc.begin_move(active)  # marks the games whose root statistics post() reads
                else:
                    mc.search(actor, active=active, waves=waves)
            finally:
                mc.set_root_noise_enabled(True)
            post()
        self._policy_only_moves = self._po_colour & (acts >= 0)
        return acts, vals

    # -- MsgRequest handling: GoGameSelfPlay::OnReceive (game_selfplay.cc:222-270) for all games ----
    def set_request(self, black_ver, white_ver=-1, black_resign_thres=None, white_resign_thres=None,
                    never_resign_prob=None, player_swap=False, async_=False, num_game_thread_used=-1):
        """Apply a server request between two moves.  Returns the reference's RestartReply name:
        ``only_wait`` (black_ver < 0: every game idles), ``update_model`` (versions or player_swap
        changed, or the games were waiting: every playing game is restarted, unfinished games are
        dropped as the reference's ``restart()`` does), ``update_model_async`` (async: the new models
        take over mid-game) or ``update_request_only`` (same versions: only thresholds change).
        ``num_game_thread_used`` >= 0 lets only the first that many games play
        (DispatcherCallback::OnFirstSend, dispatcher_callback.h:27-44)."""
        prev = self.request
        was_protocol = self.protocol
        new = {"black_ver": int(black_ver), "white_ver": int(white_ver), "player_swap": bool(player_swap),
               "async": bool(async_), "num_game_thread_used": int(num_game_thread_used)}
        is_waiting = new["black_ver"] < 0  # ModelPair::wait
        # a SelfPlay that never saw a request plays without versions; the reference's game threads
        # start out waiting -- in both cases the first real request is a (re)start
        is_prev_waiting = (prev["black_ver"] < 0) if was_protocol else True
        same_vers = (new["black_ver"], new["white_ver"]) == (prev["black_ver"], prev["white_ver"])
        same_swap = new["player_swap"] == prev["player_swap"]
        no_restart = (same_vers or new["async"]) and same_swap and not is_prev_waiting
        self.request = new
        self.protocol = True
        # GoStateExt::setRequest (go_state_ext.h:55-65)
        if black_resign_thres is not None:
            w = black_resign_thres if white_resign_thres is None else white_resign_thres
            self.resign_thres = (float(black_resign_thres) + float(w)) / 2.0
        if never_resign_prob is not None:
            self.never_resign_ratio = float(never_resign_prob)
        G = self.G
        if is_waiting:
            self.idle = np.ones(G, bool)
            return "only_wait"
        used = new["num_game_thread_used"]
        idle = np.zeros(G, bool) if used < 0 else (np.arange(G) >= used)
        was_idle = self.idle if self.idle is not None else np.zeros(G, bool)
        idle = idle | self.stopped  # slots that have played their num_games_per_thread stay out
        self.idle = idle if idle.any() else None
        if new["white_ver"] >= 0 and self.mcts2 is None:  # a match needs the second AI
            self.mcts2 = self._make_search(self._white_opts, 1)
        two = new["white_ver"] >= 0
        if not two and self.mcts2 is not None and self.actor_white is None and was_protocol:
            # back to self-play (ModelPair::is_selfplay): _ai2 is dropped
            self.mcts2.close() if hasattr(self.mcts2, "close") else None
            self.mcts2 = None
        self.swap = bool(two and new["player_swap"])
        if not no_restart:
            self.restart_games(~idle)
            return "update_model"
        # games of threads that were parked and are used again restart even if the rest carries on
        woken = was_idle & ~idle
        if woken.any():
            self.restart_games(woken)
        if not new["async"]:
            return "update_request_only"
        if self.recorders is not None:  # setAsync -> addCurrentModel: running games now span two models
            for g in np.flatnonzero(~idle):
                self.recorders[g].add_models(prev["black_ver"], prev["white_ver"], new["black_ver"], new["white_ver"])
        return "update_request_only" if same_vers else "update_model_async"

    def set_request_msg(self, msg):
        """``set_request`` from the server's MsgRequest (dict or JSON text).  The search options in
        ``vers.mcts_opt`` are recorded with the games; the running search keeps the options it was
        created with (the reference re-creates its AI from them at restart, game_selfplay.cc:165-182)."""
        from .record import parse_request

        kw, mcts_opt = parse_request(msg)
        reply = self.set_request(**kw)
        if self.recorders is not None:
            for r in self.recorders:
                r.mcts_opt = mcts_opt
        return reply

    def restart_games(self, mask):
        """GoGameSelfPlay::restart for the games in ``mask``: fresh boards and trees, no result"""
        m = np.ascontiguousarray(mask, dtype=np.uint8)
        if not m.any():
            return
        self.gb.reset(m)
        self.mcts.reset(m)
        if self.mcts2 is not None:
            self.mcts2.reset(m)
        sel = m.astype(bool)
        if self.ref is None:
            self.never_resign[sel] = self.rng.random(int(sel.sum())) < self.never_resign_ratio
        else:
            # restart(): _ai, then _ai2, are re-created -- init_ai draws their seeds from the game
            # generator in that order (game_selfplay.cc:165-182); _state_ext.restart() resets ResignCheck
            self.ref.init_actor(0, m)
            if self.mcts2 is not None:
                self.ref.init_actor(1, m)
            self._ref_started = True
            self.never_resign[sel] = False
            self._nr_drawn[sel] = False
        if self.recorders is not None:
            for g in np.flatnonzero(sel):
                self.recorders[g].restart()

    def finish_move(self, info, res=None, chosen=None):
        """everything GoGameSelfPlay::act does after the search returned (game_selfplay.cc:372-429):
        move choice and resign check on the device (``elfb200_mcts_choose``), ``GoState::forward``,
        tree advance, game end / restart.  ``info`` are the games' info words from before the search;
        ``res`` (root tables) is only needed, and fetched, when games are being recorded."""
        self._move_counter += 1
        seed = (self._seed << 20) ^ self._move_counter
        nr = self.never_resign.astype(np.uint8)
        if chosen is not None:
            acts, vals = chosen
            if self.ref is not None:  # shouldResign after every colour's choice, on the game generator
                self._resign_reference(info, acts, vals, acts != -2)
        elif self.ref is not None:
            acts, vals = self._choose_reference(info)
        else:
            acts, vals = self.mcts.choose(self.policy_distri_cutoff, self.resign_thres, nr, seed)
        if chosen is None and self.ref is None and self.mcts2 is not None:
            black = (info[:, 1] == 1) != self.swap  # games whose mover was searched by self.mcts (see phases)
            a2, v2 = self.mcts2.choose(self.policy_distri_cutoff, self.resign_thres, nr, seed)
            acts = np.where(black, acts, a2)
            vals = np.where(black, vals, v2)
        resign = acts == -1
        if self.idle is None:
            assert (acts != -2).all(), "a game was not searched"
        else:
            assert (acts[~self.idle] != -2).all(), "a game was not searched"
            assert (acts[self.idle] == -2).all()
        if self.recorders is not None:
            if res is None:
                res = self.mcts.results()
                if self.mcts2 is not None:
                    res = self.merge_results((info[:, 1] == 1) != self.swap, res, self.mcts2.results())
            for g in range(self.G):
                if acts[g] != -2:
                    po = chosen is not None and bool(self._policy_only_moves[g])  # no MCTS policy to record
                    self.recorders[g].on_move(int(info[g, 0]), int(acts[g]), None if po else res["visits"][g],
                                              float(vals[g]))
        ok = self.gb.forward(acts)
        played = ~resign if self.idle is None else (~resign & ~self.idle)
        assert ok[played].all(), "MCTS proposed an illegal move"
        self.mcts.advance(acts)
        if self.mcts2 is not None:
            self.mcts2.advance(acts)
        self.moves_played += int(played.sum())
        info2 = self.gb.info()
        done = resign | (info2[:, 9] == 1)
        if self.move_cutoff > 0:
            done |= info2[:, 0] >= self.move_cutoff
        if self.idle is not None:
            done &= ~self.idle
        if done.any():
            final = self.gb.evaluate(self.komi)
            for g in np.flatnonzero(done):
                if resign[g]:
                    fv, why = (1.0 if info[g, 1] == 2 else -1.0), "resign"
                else:
                    fv = float(final[g])
                    why = "two_pass" if info2[g, 10] else ("superko" if info2[g, 11] else "max_step")
                self.results.append((fv, int(info2[g, 0]), why))
                if self.recorders is not None:
                    q = self.request
                    self.records.append(self.recorders[g].finish(
                        fv, bool(self.never_resign[g]), model_ver=q["black_ver"], resign_thres=self.resign_thres,
                        never_resign_prob=self.never_resign_ratio, white_ver=q["white_ver"],
                        player_swap=q["player_swap"], async_=q["async"],
                        num_game_thread_used=q["num_game_thread_used"]))
            m = done.astype(np.uint8)
            self.gb.reset(m)
            self.mcts.reset(m)
            if self.mcts2 is not None:
                self.mcts2.reset(m)
            if self.ref is None:
                self.never_resign[done] = self.rng.random(int(done.sum())) < self.never_resign_ratio
            else:  # GoStateExt::restart -> ResignCheck::reset: the next game draws again at its first move
                self.never_resign[done] = False
                self._nr_drawn[done] = False
            self.games_finished += int(done.sum())
            if self.num_games_per_thread > 0:
                self.games_per_slot[done] += 1
                self.stopped |= self.games_per_slot >= self.num_games_per_thread
                if self.stopped.any():
                    self.idle = self.stopped.copy() if self.idle is None else (self.idle | self.stopped)
        return int(played.sum())
