"""Handicap stones: elfb200_place_handicap (k_place) against the compiled reference's PlaceHandicap /
GoState::applyHandicap, games continued from the handicap position through the step API, the search
from handicap roots, and the GTP commands fixed_handicap / place_free_handicap / set_free_handicap.

CPU: the kernels run on the SIMT emulator build of the kernel sources (tests/simt_emu), the online/GTP
host logic on the emulated GoBatch.  tests/test_zz_gpu_handicap.py runs the same checks on an H100."""
import ctypes

import numpy as np
import pytest
import torch

from tests import oracles

pytestmark = pytest.mark.timeout(900)


# ---- the reference's handicap entry points ---------------------------------------------------------
# PlaceHandicap (board.cc:109-126) and GoState::applyHandicap (go_state.cc:130-132) are compiled into
# oracle/_ref/libref_go{9,19}.so with the rest of the reference; they are bound here by their C++ symbol
# names.  The shim's state object is a GoState (no virtual functions, Board _board is its first member,
# go_state.h:95-226), so the state pointer is also the Board pointer PlaceHandicap takes.
_PLACE, _APPLY = "_Z13PlaceHandicapP5Boardiih", "_ZN7GoState13applyHandicapEi"


def _ref_handicap_lib(n):
    L = oracles.load_ref(n)
    f = getattr(L, _PLACE)
    f.restype, f.argtypes = ctypes.c_bool, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_ubyte]
    f = getattr(L, _APPLY)
    f.restype, f.argtypes = None, [ctypes.c_void_p, ctypes.c_int]
    return L


def ref_place_handicap(r, action):
    """PlaceHandicap(&state._board, x, y, S_BLACK) for action x*N+y; returns its verdict"""
    return bool(getattr(_ref_handicap_lib(r.n), _PLACE)(r.p, action // r.n, action % r.n, 1))


def ref_apply_handicap(r, k):
    """GoState::applyHandicap(k): the reference HandicapTable's placement of k stones"""
    getattr(_ref_handicap_lib(r.n), _APPLY)(r.p, int(k))


def ref_table_stones(n, k):
    """the stones the reference table places for k, read back from a fresh reference state"""
    r = oracles.Ref(n)
    ref_apply_handicap(r, k)
    return [int(a) for a in np.flatnonzero(r.stones() == 1)]


def need_ref(*sizes):
    for n in sizes:
        if not oracles.have_ref(n):
            pytest.skip("oracle/_ref not built")


# ---- board parity --------------------------------------------------------------------------------------
def handicap_cases(n, rng):
    """(stone list, plies played before the placement) per game: lists of different lengths (three 9x9
    games share a warp), the GTP fixed placements (and the reference table on 19x19), random free lists
    of up to 40 stones, a repeated point, every point of the board in random order (black fills the board
    until a stone would be suicide), and games that are already past ply 1"""
    from elf_b200.console import fixed_handicap_vertices
    from elf_b200.online import vertex2action

    P = n * n
    cases = [([vertex2action(v, n) for v in fixed_handicap_vertices(k, n)], 0) for k in range(2, 10)]
    if n == 19:
        cases += [(ref_table_stones(n, k), 0) for k in range(2, 10)]
    for length in (0, 1, 5, 13, 27, 40):
        cases.append(([int(a) for a in rng.choice(P, length, replace=False)], 0))
    rep = [int(a) for a in rng.choice(P, 7, replace=False)]
    cases.append((rep[:4] + [rep[1]] + rep[4:] + [rep[6]], 0))
    cases.append(([int(a) for a in rng.permutation(P)], 0))
    cases.append(([int(a) for a in rng.choice(P, 4, replace=False)], 1))
    cases.append(([int(a) for a in rng.choice(P, 6, replace=False)], 3))
    return cases


def assert_same_state(gb, refs, label, full=True, rng=None):
    n, G = gb.board_size, gb.num_games
    h, info, st, lg = gb.getHashCode(), gb.info(), gb.stones(), gb.legal_mask()
    for g, r in enumerate(refs):
        assert int(h[g]) == r.hash(), f"hash g={g} {label}"
        ri = r.info()
        ri[8] = 0  # ko_age is not part of the device state
        np.testing.assert_array_equal(info[g], ri, err_msg=f"info g={g} {label}")
        np.testing.assert_array_equal(st[g], r.stones(), err_msg=f"stones g={g} {label}")
        np.testing.assert_array_equal(lg[g, :-1], r.legal(), err_msg=f"legal g={g} {label}")
        assert lg[g, -1] == 1
    if not full:
        return
    sc, ev, e0, e1 = gb.tt_score(), gb.evaluate(7.5), gb.true_eyes(0), gb.true_eyes(1)
    d4s = range(8) if rng is None else [int(rng.integers(0, 8))]
    feats = {d4: gb.features(np.full(G, d4, np.int32)) for d4 in d4s}
    df = {d4: gb.features_df(np.full(G, d4, np.int32)) for d4 in d4s}
    for g, r in enumerate(refs):
        assert sc[g] == r.tt_score() and ev[g] == np.float32(r.evaluate(7.5)), f"score g={g} {label}"
        np.testing.assert_array_equal(e0[g], r.true_eyes(int(r.info()[1])), err_msg=f"eyes g={g} {label}")
        np.testing.assert_array_equal(e1[g], r.true_eyes(1), err_msg=f"eyes g={g} {label}")
        for d4 in d4s:
            np.testing.assert_array_equal(feats[d4][g], r.features(d4), err_msg=f"AGZ d4={d4} g={g} {label}")
            np.testing.assert_array_equal(df[d4][g], r.features_df(d4), err_msg=f"DF d4={d4} g={g} {label}")


def pick_moves(rng, refs, n):
    """per game: mostly a uniform legal non-eye move (the playout policy's candidates), sometimes a pass, an
    arbitrary (often illegal) point, or no move at all"""
    acts = np.empty(len(refs), np.int32)
    for g, r in enumerate(refs):
        u = rng.random()
        if r.terminated():
            acts[g] = n * n if u < 0.5 else int(rng.integers(0, n * n))
            continue
        cand = np.flatnonzero(r.legal() & (1 - r.true_eyes(int(r.info()[1]))))
        if u < 0.03 or len(cand) == 0:
            acts[g] = n * n
        elif u < 0.06:
            acts[g] = int(rng.integers(0, n * n))
        elif u < 0.08:
            acts[g] = -1
        else:
            acts[g] = int(rng.choice(cand))
    return acts


def run_board_parity(make_batch, n, seed, max_plies):
    """place the handicap cases on a batch and on reference states, compare everything observable, then
    play every game on from the handicap position and compare after every ply"""
    rng = np.random.default_rng(seed)
    cases = handicap_cases(n, rng)
    G = len(cases)
    gb = make_batch(G, n)
    refs = [oracles.Ref(n) for _ in range(G)]
    for t in range(max(p for _, p in cases)):  # games that have started before the placement
        acts = np.array([int(np.flatnonzero(r.legal())[7 * t + g]) if p > t else -1
                         for g, (r, (_, p)) in enumerate(zip(refs, cases))], np.int32)
        for r, a in zip(refs, acts):
            if a >= 0:
                assert r.forward(int(a))
        assert gb.forward(acts).tolist() == (acts >= 0).tolist()
    hashes_before = gb.getHashCode()
    ok = gb.place_handicap([s for s, _ in cases])
    for g, ((stones, p), r) in enumerate(zip(cases, refs)):
        want = [ref_place_handicap(r, a) for a in stones]
        assert ok[g].tolist() == want, f"accept flags g={g}"
        if p > 0:
            assert not any(want) and int(gb.getHashCode()[g]) == int(hashes_before[g])
    full = [g for g, (s, _) in enumerate(cases) if len(s) == n * n][0]
    assert not ok[full].all() and ok[full].sum() > n * n // 2  # suicide refused, the rest went on
    assert_same_state(gb, refs, "after placement")
    # at the handicap position (ply 1) the history is empty: the 16 stone planes are zero, as extractAGZ
    # finds an empty _history; then white is to move wherever a stone was accepted
    f = gb.features()
    info = gb.info()
    for g, (stones, p) in enumerate(cases):
        if p == 0:
            assert info[g, 0] == 1 and (f[g, :16] == 0).all()
            assert info[g, 1] == (2 if ok[g].any() else 1) and info[g, 4] == info[g, 5] == -1
    # a second call on the handicap position: white is to move now, the stones are still black's
    more = [[int(a) for a in rng.choice(n * n, int(rng.integers(0, 4)), replace=False)] for _ in range(G)]
    ok2 = gb.place_handicap(more)
    for g, r in enumerate(refs):
        assert ok2[g].tolist() == [ref_place_handicap(r, a) for a in more[g]], f"second placement g={g}"
    assert_same_state(gb, refs, "after the second placement")
    # the games go on from the handicap position: captures of handicap stones, ko, superko, the end
    for t in range(max_plies):
        acts = pick_moves(rng, refs, n)
        want = [r.forward(int(a)) if a >= 0 else False for r, a in zip(refs, acts)]
        np.testing.assert_array_equal(gb.forward(acts), want, err_msg=f"ok flags at ply {t}")
        assert_same_state(gb, refs, f"ply {t}", full=(t % 23 == 5), rng=rng)
        if all(r.terminated() for r in refs):
            break
    info = gb.info()
    assert info[:, 2:4].sum() > 0 and info[:, 9].any()  # there were captures, and games that ended
    gb.close()
    return t


@pytest.fixture(scope="module")
def emu():
    from tests import emu as E

    try:
        E.emu_lib()
    except Exception as e:  # no g++ / ucontext: the emulator is a convenience, not a requirement
        pytest.skip(f"SIMT emulator build unavailable: {e}")
    return E


@pytest.mark.parametrize("n,plies", [(9, 400), (19, 250)])
def test_place_handicap_matches_reference(emu, n, plies):
    need_ref(n)
    run_board_parity(emu.emu_batch, n, seed=40 + n, max_plies=plies)


def test_place_handicap_argument_checks(emu):
    from elf_b200.lib import ElfB200Error

    gb = emu.emu_batch(2, 9)
    for bad in ([[81], []], [[-1], [3]], [list(range(82)), []]):
        with pytest.raises(ElfB200Error):
            gb.place_handicap(bad)
    assert (gb.stones() == 0).all()  # a refused call places nothing
    assert [o.tolist() for o in gb.place_handicap([[], [4, 4]])] == [[], [True, False]]
    assert gb.info()[:, 1].tolist() == [1, 2]


# ---- the search from handicap positions -------------------------------------------------------------
def run_search_from_handicap(make_batch, make_search, n, stone_counts, opts, moves=3):
    """root visits, priors, chosen move and the planes of every leaf equal the compiled reference search
    (RefMcts on a reference state after PlaceHandicap) over consecutive moves with a persistent tree"""
    from elf_b200.console import fixed_handicap_vertices
    from elf_b200.online import vertex2action

    G, P1 = len(stone_counts), n * n + 1
    gb = make_batch(G, n)
    refs = [oracles.Ref(n) for _ in range(G)]
    lists = [[vertex2action(v, n) for v in fixed_handicap_vertices(k, n)] for k in stone_counts]
    assert all(o.all() for o in gb.place_handicap(lists))
    for r, s in zip(refs, lists):
        assert all(ref_place_handicap(r, a) for a in s)
    recorded = {}

    def ref_cb(feats, hashes):
        for f, h in zip(feats, hashes):
            recorded.setdefault(int(h), []).append(f.copy())
        return oracles.fakenet(hashes, P1)

    rms = [oracles.RefMcts(n, callback=ref_cb, **opts) for _ in range(G)]
    mc = make_search(gb, rotation_flip=0, **opts)
    checked = [0]

    def actor(batch):
        h, _, _ = mc.leaf_info()
        s = batch["s"].cpu().numpy()
        for i, hh in enumerate(h):
            cands = recorded.get(int(hh))
            assert cands and any((s[i] == c).all() for c in cands), f"leaf planes differ for hash {int(hh):x}"
            checked[0] += 1
        pi, v = oracles.fakenet(h, P1)
        return {"pi": torch.from_numpy(pi).to(mc.device), "V": torch.from_numpy(v).to(mc.device)}

    for mv in range(moves):
        want = [rm.act(r) for rm, r in zip(rms, refs)]  # the reference first: it fills `recorded`
        if mv == 0:  # the handicap roots: white to move, no history planes
            for g, r in enumerate(refs):
                assert int(r.info()[1]) == 2 and (recorded[r.hash()][0] == r.features(0)).all()
                assert (recorded[r.hash()][0][:16] == 0).all()
        res = mc.act(actor)
        pri = mc.root_priors()
        for g in range(G):
            np.testing.assert_array_equal(res["visits"][g], want[g]["visits"], err_msg=f"visits move {mv} game {g}")
            w = np.where(want[g]["visits"] >= 0, want[g]["prior"], -1.0).astype(np.float32)  # -1: no such edge
            np.testing.assert_array_equal(pri[g], w, err_msg=f"priors move {mv} game {g}")
            assert res["best_action"][g] == want[g]["best_action"] and res["total_visits"][g] == want[g]["total_visits"]
        acts = np.array([w["best_action"] for w in want], np.int32)
        for r, a in zip(refs, acts):
            assert r.forward(int(a))
        assert gb.forward(acts).all()
        mc.advance(acts)
    assert (mc.errors() == 0).all() and checked[0] > 0
    mc.close()
    gb.close()


SEARCH_OPTS = dict(num_rollouts=64, num_rollouts_per_batch=8, virtual_loss=1, persistent_tree=1, c_puct=1.5)


@pytest.mark.parametrize("n,stones", [(19, (2, 4, 9)), (9, (4,))])
def test_search_from_handicap_matches_reference(emu, n, stones):
    need_ref(n)
    run_search_from_handicap(emu.emu_batch, emu.EmuSearch, n, stones, SEARCH_OPTS)


# ---- online game and GTP ----------------------------------------------------------------------------
class BatchStubSearch:
    """the one-wave stub search of tests/test_online_console.py over a real (emulated) GoBatch: the move is
    the arg-max of the replied policy over the legal moves"""

    waves_per_move = 1

    def __init__(self, board):
        self.b = board
        self.advanced, self.resets = [], 0

    def begin_move(self, active):
        self.pi = self.v = None

    def select(self):
        return torch.from_numpy(self.b.features())

    def expand_backup(self, pi, v):
        self.pi, self.v = pi[0].numpy().copy(), float(v[0])

    def choose(self, cutoff, thres, never_resign, seed):
        legal = self.b.legal_mask()[0].astype(bool)
        return np.array([int(np.where(legal, self.pi, -1.0).argmax())], np.int32), np.array([self.v], np.float32)

    def advance(self, a):
        self.advanced.append(int(a[0]))

    def reset(self, mask):
        self.resets += 1


def make_console(emu, n):
    from elf_b200 import console, online

    gb = emu.emu_batch(1, n)
    g = online.OnlineGame(gb, BatchStubSearch(gb))

    def actor(batch):
        k = batch["s"].shape[0]
        pi = torch.full((k, n * n + 1), 1e-4)
        pi[:, : n * n] = torch.linspace(1.0, 0.5, n * n)  # prefers low actions: A1, A2, ...
        return {"pi": pi, "V": torch.zeros(k)}

    return g, console.GtpConsole(g, actor)


FIXED = {19: ["D4 Q16", "D4 Q16 D16", "D4 Q16 D16 Q4", "D4 Q16 D16 Q4 K10", "D4 Q16 D16 Q4 D10 Q10",
              "D4 Q16 D16 Q4 D10 Q10 K10", "D4 Q16 D16 Q4 D10 Q10 K4 K16", "D4 Q16 D16 Q4 D10 Q10 K4 K16 K10"],
         9: ["C3 G7", "C3 G7 C7", "C3 G7 C7 G3", "C3 G7 C7 G3 E5", "C3 G7 C7 G3 C5 G5", "C3 G7 C7 G3 C5 G5 E5",
             "C3 G7 C7 G3 C5 G5 E3 E7", "C3 G7 C7 G3 C5 G5 E3 E7 E5"]}


def _black_vertices(g):
    from elf_b200 import online

    st = g.board.stones()[0]
    return sorted(online.action2vertex(int(a), g.N) for a in np.flatnonzero(st == 1))


@pytest.mark.parametrize("n", [9, 19])
@pytest.mark.parametrize("cmd", ["fixed_handicap", "place_free_handicap"])
def test_gtp_fixed_handicap(emu, n, cmd):
    g, c = make_console(emu, n)
    for k in range(2, 10):
        assert c.execute(f"clear_board") == "=\n\n"
        assert c.execute(f"{cmd} {k}") == f"= {FIXED[n][k - 2]}\n\n"
        assert _black_vertices(g) == sorted(FIXED[n][k - 2].split()) and (g.board.stones()[0] != 2).all()
        pic = c.execute("showboard")
        assert pic.count("X") == k + 1 and "nextPlayer: White" in pic  # k stones + the "BLACK (X)" caption
        assert g.info()[0] == 1 and g.getNextPlayer() == "W"
    assert g.finished == [] and g.seq == 0  # clearing a handicap position finishes no game


def test_gtp_handicap_game_and_errors(emu):
    from elf_b200 import online

    n = 9
    g, c = make_console(emu, n)
    empty = lambda: not g.board.stones()[0].any() and g.info()[0] == 1 and g.getNextPlayer() == "B"  # noqa: E731
    for line in ("fixed_handicap 1", "fixed_handicap 10", "fixed_handicap x", "fixed_handicap", "place_free_handicap 0"):
        assert c.execute(line) == "? invalid number of stones\n\n" and empty(), line
    for line in ("set_free_handicap", "set_free_handicap C3", "set_free_handicap C3 C3", "set_free_handicap C3 pass",
                 "set_free_handicap C3 K10", "set_free_handicap C3 J10", "set_free_handicap C3 X", "set_free_handicap C3 Q"):
        assert c.execute(line) == "? bad vertex list\n\n" and empty(), line
    # a stone the board refuses (the last point of a board filled with black) leaves the board empty
    every = " ".join(online.action2vertex(a, n) for a in range(n * n))
    assert c.execute("set_free_handicap " + every) == "? bad vertex list\n\n" and empty()
    assert g.search.resets == 0
    # a handicap game: white is to move, black may not
    assert c.execute("set_free_handicap C3 G7 E5") == "=\n\n" and g.search.resets == 1
    assert _black_vertices(g) == ["C3", "E5", "G7"]
    for cmd in ("fixed_handicap 2", "place_free_handicap 2", "set_free_handicap A1 A2"):
        assert c.execute(cmd) == "? board not empty\n\n"
    assert c.execute("genmove b").startswith("? Specified next player b is not the same as the next player W")
    assert c.execute("play b A1").startswith("? Specified next player b")
    assert c.execute("play w A1") == "=\n\n" and g.info()[0] == 2
    assert c.execute("genmove b") == "= A2\n\n" and g.info()[0] == 3  # the stub's first free preference
    assert c.execute("fixed_handicap 2") == "? board not empty\n\n"
    # clearing a started handicap game finishes it, as any started game
    assert c.execute("clear_board") == "=\n\n" and empty() and g.finished[-1][1:] == (3, "clear")
    # a passed game is not empty either
    assert c.execute("play b pass") == "=\n\n" and c.execute("fixed_handicap 2") == "? board not empty\n\n"
    assert c.execute("clear_board") == "=\n\n" and empty()
    for cmd in ("fixed_handicap", "place_free_handicap", "set_free_handicap"):
        assert c.execute(f"known_command {cmd}") == "= true\n\n"
        assert cmd in c.execute("list_commands").split()


def test_online_place_handicap(emu):
    g, _ = make_console(emu, 9)
    assert g.place_handicap([20, 60]) and g.search.resets == 1
    assert not g.place_handicap([30])  # not empty any more
    g.human(-97)  # SA_CLEAR
    assert not g.board.stones()[0].any() and g.finished == [] and g.search.resets == 2
    assert not g.place_handicap([20, 20]) and not g.board.stones()[0].any()  # refused stone: nothing stays
    assert g.search.resets == 2 and g.getNextPlayer() == "B"


def test_console_without_handicap_support():
    """a board that cannot take handicap stones does not offer the commands"""
    from elf_b200 import console, online
    from tests.test_online_console import StubBoard, StubSearch

    b = StubBoard(9, oracles.load_oracle())
    c = console.GtpConsole(online.OnlineGame(b, StubSearch(b)), None)
    assert not set(console.HANDICAP_COMMANDS) & set(c.commands)
    assert c.execute("fixed_handicap 2") == "? unknown command\n\n"
