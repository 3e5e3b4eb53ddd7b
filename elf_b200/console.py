"""GTP console over an OnlineGame -- the reference's ``df_console.py`` without the C++ game thread.

Reference: ``scripts/elfgames/go/console_lib.py:216-372`` (class GoConsoleGTP: the ``on_<command>``
table, ``check_player``, the ``= msg`` / ``? msg`` replies) and ``scripts/elfgames/go/
df_console.py:18-82`` (wiring: ``human_actor`` -> ``console.prompt``, ``actor_black`` -> evaluator).

Command set and behaviour follow the reference: ``protocol_version name version list_commands
known_command boardsize komi clear_board play genmove showboard final_score quit exit``;
``play`` / ``genmove`` refuse a colour that is not the side to move; ``boardsize`` / ``komi`` only
accept the values the engine was created with; ``final_score`` reports the value of the last
finished game (``getLastScore``), as the reference does.  Replies use the GTP wire format
(``= text\\n\\n`` / ``? text\\n\\n``, optional numeric command id echoed).

Beyond ``console_lib.py``, three GTP 2 commands start a handicap game: ``fixed_handicap n`` and
``place_free_handicap n`` (2 <= n <= 9; both place the GTP fixed placement and reply with its vertices) and
``set_free_handicap v1 v2 ...``.  They need an empty board and a board that can take handicap stones
(``GoBatch.place_handicap``); afterwards white is to move.

``final_status_list alive|dead|seki`` (GTP 2) lists the groups of the position the game ended in, one group
per line (vertices ascending, groups by their lowest vertex).  Dead groups come from Monte-Carlo ownership
(``OnlineGame.final_status``: 1024 random playouts from the position); ``seki`` is always empty, there is no
seki detection.  It is offered when the board behind the game can play those playouts
(``GoBatch.ownership``).

The reference console talks to its game thread by returning special actions from the
``human_actor`` callback; here the same special actions go straight into ``OnlineGame.human``.
(The unmodified reference console can also be run against this engine through
``elf_b200.compat.OnlineEngine``.)
"""
import sys

from . import online as _o

HANDICAP_COMMANDS = ("fixed_handicap", "place_free_handicap", "set_free_handicap")


def fixed_handicap_vertices(n, board_size):
    """the GTP 2 fixed placement of ``n`` (2..9) handicap stones: 19x19 on the 4-4 points and their
    midpoints (D4 Q16 D16 Q4, D10 Q10, K4 K16, K10), 9x9 by the same rule on the 3-3 points"""
    lo = 3 if board_size >= 13 else 2
    hi, mid = board_size - 1 - lo, board_size // 2
    xy = [(lo, lo), (hi, hi), (lo, hi), (hi, lo)][: min(n, 4)]
    if n >= 6:
        xy += [(lo, mid), (hi, mid)]
    if n >= 8:
        xy += [(mid, lo), (mid, hi)]
    if n >= 5 and n % 2 == 1:
        xy.append((mid, mid))
    return [_o.xy2move(x, y) for x, y in xy]


class GtpConsole:
    def __init__(self, game, actor, name="DF2", version="1.0"):
        self.game = game
        self.actor = actor
        self.name = name
        self.version = version
        self.board_size = game.N
        self.exit = False
        self.commands = {k[3:]: getattr(self, k) for k in dir(self) if k.startswith("on_")}
        if getattr(game.board, "place_handicap", None) is None:  # a board that cannot take handicap stones
            for k in HANDICAP_COMMANDS:
                del self.commands[k]
        if getattr(game.board, "ownership", None) is None:  # a board that cannot play ownership playouts
            del self.commands["final_status_list"]
        self.final_status_playouts = 1024

    # -- helpers ---------------------------------------------------------------------------------
    def check_player(self, player):  # console_lib.py:313-325
        board_next = self.game.getNextPlayer()
        if player.lower() != board_next.lower():
            return False, ("Specified next player %s is not the same as the next player %s on the board"
                           % (player, board_next))
        return True, None

    def move2action(self, v):  # console_lib.py:289-294
        special = {"skip": _o.SA_SKIP, "pass": _o.SA_PASS, "resign": _o.SA_RESIGN, "clear": _o.SA_CLEAR}
        if v.lower() in special:
            return special[v.lower()]
        return _o.vertex2action(v, self.board_size)

    # -- commands: (ok, text) ----------------------------------------------------------------------
    def on_protocol_version(self, items):
        return True, "2"

    def on_name(self, items):
        return True, self.name

    def on_version(self, items):
        return True, self.version

    def on_list_commands(self, items):
        return True, "\n".join(sorted(self.commands))

    def on_known_command(self, items):
        return True, "true" if len(items) > 1 and items[1] in self.commands else "false"

    def on_boardsize(self, items):
        if items[1] != str(self.board_size):
            return False, "We only support %dx%d board for now" % (self.board_size, self.board_size)
        return True, ""

    def on_komi(self, items):
        if float(items[1]) != self.game.komi:
            return False, "We only support %s komi for now" % self.game.komi
        return True, ""

    def on_clear_board(self, items):
        self.game.human(_o.SA_CLEAR)
        return True, ""

    def on_play(self, items):
        ok, msg = self.check_player(items[1][0])
        if not ok:
            return False, msg
        st = self.game.human(self.move2action(items[2]))
        if st == _o.INVALID:
            return False, "illegal move"
        return True, ""

    def on_genmove(self, items):
        ok, msg = self.check_player(items[1][0])
        if not ok:
            return False, msg
        st = self.game.human(_o.SA_SKIP)
        if st == _o.FINISHED:  # the position was already terminal
            return True, "PASS"
        a = self.game.genmove(self.actor)
        if a == _o.SA_RESIGN:
            return True, "resign"
        if a is None:
            return True, "PASS"
        return True, _o.action2vertex(a, self.board_size)

    def on_showboard(self, items):
        return True, "\n" + self.game.showBoard().rstrip("\n")

    # -- handicap (GTP 2 section 6.3.2) -----------------------------------------------------------
    def _board_empty(self):
        return int(self.game.info()[0]) == 1 and not self.game.board.stones()[0].any()

    def on_fixed_handicap(self, items):
        if not self._board_empty():
            return False, "board not empty"
        try:
            n = int(items[1])
        except (IndexError, ValueError):
            n = 0
        if not 2 <= n <= 9:
            return False, "invalid number of stones"
        vs = fixed_handicap_vertices(n, self.board_size)
        if not self.game.place_handicap([_o.vertex2action(v, self.board_size) for v in vs]):
            return False, "board not empty"
        return True, " ".join(vs)

    on_place_free_handicap = on_fixed_handicap  # the engine may choose any placement: the fixed one

    def on_set_free_handicap(self, items):
        if not self._board_empty():
            return False, "board not empty"
        acts = []
        for v in items[1:]:
            try:
                a = _o.vertex2action(v, self.board_size)
            except ValueError:  # off the board, or not a vertex
                return False, "bad vertex list"
            if a == self.board_size * self.board_size or a in acts:
                return False, "bad vertex list"
            acts.append(a)
        if len(acts) < 2 or not self.game.place_handicap(acts):  # a stone the board refuses: nothing placed
            return False, "bad vertex list"
        return True, ""

    # -- end of game (GTP 2 section 6.3.5) ---------------------------------------------------------
    def on_final_status_list(self, items):
        status = items[1].lower() if len(items) > 1 else ""
        if status not in ("alive", "dead", "seki"):
            return False, "syntax error"
        if status == "seki":  # no seki detection
            return True, ""
        dead, alive = self.game.final_status(playouts=self.final_status_playouts)
        groups = dead if status == "dead" else alive
        return True, "\n".join(" ".join(_o.action2vertex(a, self.board_size) for a in g) for g in groups)

    def on_final_score(self, items):
        s = self.game.getLastScore()
        return True, ("B+%.1f" % s) if s > 0 else ("W+%.1f" % (-s))

    def on_quit(self, items):
        self.exit = True
        return True, ""

    on_exit = on_quit

    # -- the loop ----------------------------------------------------------------------------------
    def execute(self, line):
        """one GTP command line -> the full reply text ('' for blank lines / comments)"""
        line = line.split("#", 1)[0].strip()
        if not line:
            return ""
        items = line.split()
        cid = ""
        if items[0].isdigit():
            cid = items.pop(0)
            if not items:
                return "?%s empty command\n\n" % cid
        try:
            fn = self.commands.get(items[0])
            if fn is None:
                ok, msg = False, "unknown command"
            else:
                ok, msg = fn(items)
        except Exception as e:  # the reference prints the traceback and answers "? Invalid command"
            ok, msg = False, "Invalid command (%s)" % e
        return "%s%s %s\n\n" % ("=" if ok else "?", cid, msg) if msg else "%s%s\n\n" % ("=" if ok else "?", cid)

    def run(self, inp=None, out=None):
        inp = inp or sys.stdin
        out = out or sys.stdout
        for line in inp:
            r = self.execute(line)
            if r:
                out.write(r)
                out.flush()
            if self.exit:
                break
