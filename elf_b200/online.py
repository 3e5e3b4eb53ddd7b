"""OnlineGame: the single-game "online" mode of the reference's game loop on top of the GPU engine.

Reference: ``GoGameSelfPlay`` with ``mode == "online"`` (``src_cpp/elfgames/go/common/
game_selfplay.cc:186-219`` restart + SGF preload, ``:293-330`` the human branch of ``act``,
``:350-437`` the AI branch, ``:121-149`` finish_game) and ``GoStateExt`` (``common/
go_state_ext.h:79-118,207-214``: final value, last move of the finished game, resign rule).

One board (a ``GoBatch`` of one game) and one search (``MctsBatch``) are driven by two entry points:

* ``human(action)``  -- what the reference does with the reply of the ``human_actor`` label: a board
  action ``x*N+y`` / ``N*N`` (pass), or one of the special actions ``SA_SKIP`` (let the AI move),
  ``SA_PASS``, ``SA_RESIGN``, ``SA_CLEAR`` (``common/game_feature.h:17,50-66``);
* ``genmove(actor)`` -- the AI branch: one MCTS, most visited move (or a sample while
  ``ply <= policy_distri_cutoff``), resign rule, optional SGF following, ``forward``, tree advance,
  game end.  ``ai_search()`` is the same search as a generator cut at every network round trip, for
  callers that own the network loop (``elf_b200.compat.OnlineEngine``).

``board`` and ``search`` are duck-typed (``GoBatch`` / ``MctsBatch`` interfaces) so the host logic can
be exercised without a GPU by the CPU tests; ``OnlineGame.create`` builds the real ones.
"""
import numpy as np

from . import sgf as _sgf

SA_SKIP, SA_PASS, SA_RESIGN, SA_CLEAR = -100, -99, -98, -97  # SpecialActionType, game_feature.h:17
S_BLACK, S_WHITE = 1, 2

# what human() reports back
MOVED, INVALID, SKIP, CLEARED, RESIGNED, FINISHED = "moved", "invalid", "skip", "cleared", "resigned", "finished"

_GTP_COLS = "ABCDEFGHJKLMNOPQRSTUVWXYZ"  # no 'I'


def move2xy(v):
    """GTP vertex -> (x, y); "pass" -> (-1, -1)   (scripts/elfgames/go/console_lib.py:12-20)"""
    if v.lower() == "pass":
        return -1, -1
    x = ord(v[0].lower()) - ord("a")
    if x >= 9:  # skip 'i'
        x -= 1
    return x, int(v[1:]) - 1


def xy2move(x, y):
    """(x, y) -> GTP vertex   (console_lib.py:23-29)"""
    if x == -1 and y == -1:
        return "pass"
    return _GTP_COLS[x] + str(y + 1)


def vertex2action(v, n):
    x, y = move2xy(v)
    if x == -1:
        return n * n
    if not (0 <= x < n and 0 <= y < n):
        raise ValueError(f"vertex {v} is off the {n}x{n} board")
    return x * n + y


def action2vertex(a, n):
    """coord2str2 (sgf/sgf.h:73-86): what getLastMove() prints"""
    if a == n * n:
        return "PASS"
    if a == SA_RESIGN:
        return "RESIGN"
    if a is None or a < 0:
        return ""
    return _GTP_COLS[a // n] + str(a % n + 1)


def _star(n, i, j):  # STAR_ON9 / 13 / 19, base/board.h:16-27
    if n == 19:
        return i in (3, 9, 15) and j in (3, 9, 15)
    if n == 13:
        return (i in (3, 9) and j in (3, 9)) or (i == 6 and j == 6)
    if n == 9:
        return (i in (2, 6) and j in (2, 6)) or (i == 4 and j == 4)
    return False


def show_board(stones, n, last_action, b_cap, w_cap, next_player):
    """GoState::showBoard (base/go_state.h:187-192) = showBoard2Buf(SHOW_LAST_MOVE)
    (base/board.cc:1414-1459) + the last-move / next-player line.  ``stones``: uint8[N*N] by action."""
    prompt = " ".join(_GTP_COLS[:n])
    out = ["   " + prompt + "\n"]
    for j in range(n - 1, -1, -1):
        row = "%2d " % (j + 1)
        for i in range(n):
            a = i * n + j
            s = int(stones[a])
            if s in (S_BLACK, S_WHITE):
                ch = "X" if s == S_BLACK else "O"
                row += ch + (")" if a == last_action else " ")
            else:
                row += "+ " if _star(n, i, j) else ". "
        row += "%d" % (j + 1)
        if j == n // 2 + 1:
            row += "     WHITE (O) has captured %d stones" % w_cap
        elif j == n // 2:
            row += "     BLACK (X) has captured %d stones" % b_cap
        out.append(row + "\n")
    out.append("   " + prompt)
    # before the first move the reference prints coord2str2(M_INVALID) = "C0" (M_INVALID is the
    # off-board coordinate (2,-1), base/common.h); kept so the picture is byte-identical
    last = action2vertex(last_action, n) if last_action is not None and last_action >= 0 else "C0"
    return "".join(out) + "\nLast move: " + last + ", nextPlayer: " + ("Black" if next_player == S_BLACK else "White") + "\n"


def stone_groups(stones, n):
    """the groups (4-connected stones of one colour) of a position given as colours by action x*N+y: lists of
    actions in ascending order, ordered by their lowest action"""
    seen = np.zeros(n * n, bool)
    groups = []
    for a in range(n * n):
        if stones[a] == 0 or seen[a]:
            continue
        grp, todo = [], [a]
        seen[a] = True
        while todo:
            p = todo.pop()
            grp.append(p)
            x, y = divmod(p, n)
            for q in ((p - n) if x > 0 else -1, (p + n) if x < n - 1 else -1, (p - 1) if y > 0 else -1,
                      (p + 1) if y < n - 1 else -1):
                if q >= 0 and not seen[q] and stones[q] == stones[a]:
                    seen[q] = True
                    todo.append(q)
        groups.append(sorted(grp))
    return groups


class OnlineGame:
    def __init__(self, board, search, komi=7.5, resign_thres=0.0, policy_distri_cutoff=0, move_cutoff=-1,
                 preload_sgf=None, preload_sgf_move_to=-1, following_pass=False, seed=0):
        if board.num_games != 1:
            raise ValueError("OnlineGame drives exactly one game")
        self.board = board
        self.search = search
        self.N = board.board_size
        self.komi = float(komi)
        self.resign_thres = float(resign_thres)
        self.policy_distri_cutoff = int(policy_distri_cutoff)
        self.move_cutoff = int(move_cutoff)
        self.following_pass = bool(following_pass)
        self._seed = int(seed)
        self._moves = 0
        self.last_value = 0.0  # GoStateExt::_last_value: final value of the last finished game
        self._last_move_of_finished = None  # GoStateExt::_last_move_for_the_game
        self.seq = 0
        self.finished = []  # (final_value, plies, reason) per finished game
        self._sgf = None
        self._sgf_pos = 0
        self._preload = (preload_sgf, int(preload_sgf_move_to))
        self._final = None  # one-game batch holding the position of the last finished game
        self._final_kept = False
        self._restart(first=True)

    @classmethod
    def create(cls, board_size=19, device=0, komi=7.5, **kw):
        """the real thing: a GoBatch of one game + its MctsBatch (keyword arguments that name an
        ``elfb200_mcts_options`` field go to the search, the rest to OnlineGame)"""
        from . import lib as _l
        from .board import GoBatch
        from .mcts import MctsBatch

        mcts_fields = {f[0] for f in _l.MctsOptions._fields_}
        mo = {k: kw.pop(k) for k in list(kw) if k in mcts_fields}
        mo.setdefault("komi", komi)
        gb = GoBatch(1, board_size=board_size, device=device)
        return cls(gb, MctsBatch(gb, **mo), komi=komi, **kw)

    # -- observers (GoGameSelfPlay::showBoard/getNextPlayer/getLastMove/getScore/getLastScore,
    #    common/game_selfplay.h:41-56) ---------------------------------------------------------
    def info(self):
        return self.board.info()[0]

    def showBoard(self):
        i = self.info()
        return show_board(self.board.stones()[0], self.N, int(i[4]), int(i[2]), int(i[3]), int(i[1]))

    def getNextPlayer(self):
        return "B" if int(self.info()[1]) == S_BLACK else "W"  # player2str, sgf.h:59-71

    def last_action(self):
        """GoStateExt::lastMove (go_state_ext.h:107-112): right after a restart, the last move of the
        game that just ended"""
        i = self.info()
        if int(i[0]) == 1:  # justStarted
            return self._last_move_of_finished
        return int(i[4])

    def getLastMove(self):
        return action2vertex(self.last_action(), self.N)

    def getScore(self):
        return float(self.board.evaluate(self.komi)[0])

    def getLastScore(self):
        return self.last_value

    # -- game boundaries -------------------------------------------------------------------------
    def _restart_game(self):
        """what finish_game does at the end (game_selfplay.cc:121-149: _ai->endGame + _state_ext.restart()):
        an empty board and tree.  The SGF preload is NOT repeated and the SGF iterator stays where it
        was -- both belong to GoGameSelfPlay::restart(), which only runs when a request arrives."""
        self.board.reset(None)
        self.search.reset(None)
        self.seq += 1

    def _restart(self, first=False):
        """GoGameSelfPlay::restart (game_selfplay.cc:186-219): fresh state, then the SGF preload"""
        if not first:
            self._restart_game()
        path, move_to = self._preload
        if path:  # game_selfplay.cc:202-219
            self._sgf = _sgf.Sgf.load(path, self.N) if isinstance(path, str) else path
            self._sgf_pos = 0
            while self._sgf_pos < len(self._sgf.moves) and self._sgf_pos < move_to:
                a = self._sgf.moves[self._sgf_pos].action
                if a < 0 or not self._forward(a):
                    raise RuntimeError("Preload sgf: move not valid!")
                self._sgf_pos += 1

    def _forward(self, a):
        ok = bool(self.board.forward(np.array([a], np.int32))[0])
        if ok:
            self.search.advance(np.array([a], np.int32))
        return ok

    def _finish_game(self, reason):
        """finish_game (game_selfplay.cc:121-149) + GoStateExt::setFinalValue / restart"""
        i = self.info()
        if reason == "resign":
            fv = 1.0 if int(i[1]) == S_WHITE else -1.0  # the side to move resigns
            self._last_move_of_finished = SA_RESIGN
        else:
            fv = self.getScore()
            self._last_move_of_finished = int(i[4])
        self.last_value = fv
        self.finished.append((fv, int(i[0]), reason))
        self._keep_final_position()
        self._restart_game()
        return fv

    def _keep_final_position(self):
        """copy the finished position into a one-game batch before the restart, so ``final_status`` can still
        look at it (boards that cannot copy games keep nothing)"""
        if getattr(self.board, "gather", None) is None:
            return
        if self._final is None:
            self._final = self.board.new_like(1)
        self._final.gather(self.board, [0])
        self._final_kept = True

    # -- end of game: dead stones -------------------------------------------------------------------
    def final_status(self, playouts=1024, seed=0, threshold=0.5):
        """dead and alive groups of the position the game ended in: the kept final position when the board
        was restarted after a finished game and nothing has been played since, the current position otherwise.
        A group is dead when ``playouts`` random playouts from the position leave its stones, on average, more
        than ``threshold`` in the opponent's area (``GoBatch.ownership`` / ``GoBatch.final_status``).  Returns
        ``(dead, alive)``: lists of groups, each a list of actions (x*N+y) in ascending order, the groups
        ordered by their lowest action."""
        board = self.board
        i = self.info()
        if self._final_kept and int(i[0]) == 1 and not board.stones()[0].any():
            board = self._final
        counts = board.ownership(playouts, seed=seed)
        dead = board.final_status(counts, playouts, threshold)[0][0]
        dead_groups, alive_groups = [], []
        for grp in stone_groups(board.stones()[0], self.N):
            (dead_groups if dead[grp[0]] else alive_groups).append(grp)
        return dead_groups, alive_groups

    # -- handicap -----------------------------------------------------------------------------------
    def place_handicap(self, actions):
        """GoState::applyHandicap on the game about to start: black stones at ``actions`` (x*N+y), each
        placed as PlaceHandicap does (board.cc:109-126); afterwards white is to move and the ply is still 1.
        Only on an empty board at ply 1.  If the board refuses any stone it is emptied again, so it never
        holds part of a setup.  Returns True when all stones are on the board."""
        i = self.info()
        if int(i[0]) != 1 or self.board.stones()[0].any():
            return False
        ok = self.board.place_handicap([[int(a) for a in actions]])[0]
        if not ok.all():
            self.board.reset(None)
            return False
        self.search.reset(None)  # the tree's root is the empty board: it no longer matches (DESIGN 3 (ii))
        return True

    # -- the human branch of act() ----------------------------------------------------------------
    def human(self, action):
        i = self.info()
        if int(i[9]):  # s.terminated()
            self._finish_game("illegal")
            return FINISHED
        action = int(action)
        if action == SA_SKIP:
            return SKIP
        if action == SA_CLEAR:
            if int(i[0]) != 1:  # !justStarted
                self._finish_game("clear")
            elif self.board.stones()[0].any():  # handicap stones, still ply 1: no game to finish
                self.board.reset(None)
                self.search.reset(None)
            return CLEARED
        if action == SA_RESIGN:
            self._finish_game("resign")
            return RESIGNED
        if action == SA_PASS:
            action = self.N * self.N
        if not (0 <= action <= self.N * self.N) or not self._forward(action):
            return INVALID  # "Invalid move ... please try again"
        if int(self.info()[10]):  # isTwoPass: "If the human opponent pass, we pass as well"
            self._finish_game("two_pass")
            return FINISHED
        return MOVED

    # -- the AI branch of act() -------------------------------------------------------------------
    def ai_search(self):
        """generator: yields the leaf feature tensor of every wave that needs the network and
        expects ``(pi, V)`` back through ``send``; returns when the search is complete"""
        mc = self.search
        mc.begin_move(None)
        for _ in range(mc.waves_per_move):
            s = mc.select()
            if s.shape[0] > 0:
                self.board.synchronize()
                pi, v = yield s
                mc.expand_backup(pi, v)
            else:
                mc.expand_backup(None, None)

    def ai_finish(self):
        """everything after the search (game_selfplay.cc:372-437); returns the action played,
        SA_RESIGN, or None when the game ended without a move (SGF exhausted)"""
        self._moves += 1
        acts, vals = self.search.choose(self.policy_distri_cutoff, self.resign_thres, None,
                                        (self._seed << 20) ^ self._moves)
        a = int(acts[0])
        if self.following_pass and a >= 0:
            # mcts_update_info (game_selfplay.cc:97-119): the opponent passed and we are clearly ahead
            # (score on the board and predicted value agree) -> pass as well
            i = self.info()
            v, score = float(vals[0]), self.getScore()
            good = (score > 0 and v > 0.9) if int(i[1]) == S_BLACK else (score < 0 and v < -0.9)
            if good and int(i[4]) == self.N * self.N:
                a = self.N * self.N
        if a == -1:  # shouldResign && ply >= 50
            self._finish_game("resign")
            return SA_RESIGN
        if self._sgf is not None and self._sgf.num_moves > 0:  # follow the preloaded record
            if self._sgf_pos >= len(self._sgf.moves):
                self._finish_game("max_step")
                return None
            a = self._sgf.moves[self._sgf_pos].action
            self._sgf_pos += 1
        if a < 0 or not self._forward(a):
            raise RuntimeError(f"Something is wrong! Move {a} cannot be applied")
        i = self.info()
        if int(i[9]):
            self._finish_game("two_pass" if int(i[10]) else ("illegal" if int(i[11]) else "max_step"))
        elif self.move_cutoff > 0 and int(i[0]) >= self.move_cutoff:
            self._finish_game("max_step")
        return a

    def genmove(self, actor):
        """MCTSGoAI::act + the rest of the AI branch with ``actor(batch) -> {"pi", "V"}``"""
        import torch

        if int(self.info()[9]):
            self._finish_game("illegal")
            return None
        gen = self.ai_search()
        try:
            s = next(gen)
            while True:
                with torch.no_grad():
                    reply = actor({"s": s})
                pi = reply["pi"].to(torch.float32).contiguous()
                v = reply["V"].to(torch.float32).reshape(-1).contiguous()
                if pi.is_cuda:
                    torch.cuda.current_stream(pi.device).synchronize()
                s = gen.send((pi, v))
        except StopIteration:
            pass
        return self.ai_finish()
