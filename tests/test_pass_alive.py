"""Pass-alive chains and areas (elfb200_pass_alive / elfb200_pass_alive_dev, k_pass_alive, GoBatch.pass_alive) and the
pass-alive dead-stone rule (elfb200_final_status_pass_alive, k_final_status<N, true>, GoBatch.final_status(
pass_alive=True), OnlineGame.final_status, GTP final_status_list) against tests/benson_ref.py, a plain restatement of
the definition in include/elfb200.h.  The reference has no counterpart to the analysis; territory and score are
checked against its getTrompTaylorScore with the dead set, as tests/test_ownership.py binds it.

CPU: the kernels run on the SIMT emulator build of the kernel sources (tests/simt_emu) under every lane order.
tests/test_zz_gpu_pass_alive.py runs the checks at full batch size on an H100."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import benson_ref as B
from tests import oracles

pytestmark = pytest.mark.timeout(900)

ERR_ARG = -1  # ELFB200_ERR_ARG (include/elfb200.h)


# ---- positions -----------------------------------------------------------------------------------------------
def setup_moves(black, white, n):
    """a move list that places the stones: black and white alternate, a pass where one colour has none left (never
    two passes in a row), a trailing pass dropped"""
    P = n * n
    b, w = list(black), list(white)
    mv = []
    while b or w:
        mv.append(b.pop(0) if b else P)
        mv.append(w.pop(0) if w else P)
    while mv and mv[-1] == P:
        mv.pop()
    return mv


def d4(x, y, n, t):
    """the t-th (0..7) symmetry of the square applied to point (x, y)"""
    if t & 4:
        x, y = y, x
    if t & 1:
        x = n - 1 - x
    if t & 2:
        y = n - 1 - y
    return x, y


# Hand-built positions in the corner: rows y, columns x; X black, O white.  The expected answer uses A for an
# alive stone, b / w for a point of black's / white's area, '.' for neither.
HAND = [
    ("two one-point eyes in the corner",
     [".X.X",
      "XXXX"],
     ["bAbA",
      "AAAA"]),
    ("one eye, the rest open",
     [".X",
      "XX"],
     ["..",
      ".."]),
    # Benson's shared eyes: chains (1,0)-(2,0)-(2,1) and (0,1)-(0,2)-(1,2); each one-point region touches both
    ("two chains sharing two one-point eyes",
     [".XX",
      "X.X",
      "XX."],
     ["bAA",
      "AbA",
      "AA."]),
    # the enclosed six points are not all liberties of the chain: only the eye is vital to it
    ("one eye and a large enclosed region that is not vital",
     [".X...X",
      "XX...X",
      ".XXXXX"],
     ["......",
      "......",
      "......"]),
    # the inner black (1,0)-(2,0)-(2,1) and white (0,1)-(0,2)-(1,2) chains share their three liberties
    ("seki",
     [".XXO",
      "O.XO",
      "OO.O",
      "XXX."],
     ["....",
      "....",
      "....",
      "...."]),
    ("an opponent stone inside an eye region",
     [".X.O.X",
      "XXXXXX"],
     ["bAbbbA",
      "AAAAAA"]),
    ("a single stone",
     ["X"],
     ["."]),
    ("the empty board",
     [],
     []),
]


def filled_board(n):
    """black on every point but spread one-point eyes: every point is alive or black's area"""
    eyes = {(1, 1), (n - 2, n - 2), (1, n - 2), (n - 2, 1), (n // 2, n // 2)}
    black = [x * n + y for x in range(n) for y in range(n) if (x, y) not in eyes]
    exp_alive = np.zeros(n * n, np.uint8)
    exp_alive[black] = 1
    exp_area = np.zeros(n * n, np.uint8)
    exp_area[[x * n + y for x, y in eyes]] = 1
    return black, exp_alive, exp_area


def hand_case(case, n, t, swap):
    """(black, white, expected alive, expected area) of a hand-built case under symmetry t, colours swapped"""
    _, pos, exp = case
    black, white = [], []
    alive, area = np.zeros(n * n, np.uint8), np.zeros(n * n, np.uint8)
    for y, (row, erow) in enumerate(zip(pos, exp)):
        for x, (c, e) in enumerate(zip(row, erow)):
            tx, ty = d4(x, y, n, t)
            a = tx * n + ty
            if c != ".":
                (black if (c == "X") != swap else white).append(a)
            if e == "A":
                alive[a] = 1
            elif e in "bw":
                area[a] = 1 if (e == "b") != swap else 2
    return black, white, alive, area


def all_hand_cases(n):
    """(name, move list, expected alive, expected area) of every hand-built case, symmetry and colour"""
    out = []
    for case in HAND:
        for t in range(8):
            for swap in (False, True):
                b, w, al, ar = hand_case(case, n, t, swap)
                out.append((f"{case[0]} (d4 {t}{', colours swapped' if swap else ''})", setup_moves(b, w, n), b, w,
                            al, ar))
    b, al, ar = filled_board(n)
    out.append(("black filled the board but one-point eyes", setup_moves(b, [], n), b, [], al, ar))
    return out


def eye_avoiding_game(n, rng, lib=None, max_plies=None):
    """a game of the eye-avoiding random policy on the C restatement (tests/oracles.Oracle): each ply a uniformly
    chosen legal move that is not one of the mover's own true eyes, a pass when there is none, until the game ends
    (or after max_plies plies); the moves"""
    o = oracles.Oracle(n, lib=lib)
    moves = []
    while not o.terminated() and (max_plies is None or len(moves) < max_plies):
        me = int(o.info()[1])
        cand = np.flatnonzero(o.legal() & (1 - o.true_eyes(me)))
        a = int(rng.choice(cand)) if len(cand) else n * n
        assert o.forward(a)
        moves.append(a)
    return moves, o.stones()


def corpus_chunk(args):
    """(move lists, stones, expected alive, expected area) of `count` games; max_plies None: terminal positions"""
    n, seed, count, max_plies = args
    rng = np.random.default_rng(seed)
    lists, st, al, ar = [], [], [], []
    for _ in range(count):
        mv, s = eye_avoiding_game(n, rng, max_plies=max_plies)
        a, r = B.benson(s, n)
        lists.append(mv)
        st.append(s)
        al.append(a)
        ar.append(r)
    return lists, np.array(st, np.uint8), np.array(al, np.uint8), np.array(ar, np.uint8)


# ---- checks --------------------------------------------------------------------------------------------------
def check_invariants(stones, alive, area):
    assert not (alive.astype(bool) & (stones == 0)).any()  # alive only on stones
    assert not ((area == 1) & (stones == 1)).any() and not ((area == 2) & (stones == 2)).any()
    assert not ((area == 1) & (alive == 1) & (stones == 2)).any()  # a white alive stone in black's area
    assert not ((area == 2) & (alive == 1) & (stones == 1)).any()
    assert set(np.unique(area)) <= {0, 1, 2} and set(np.unique(alive)) <= {0, 1}


def run_equal_restatement(gb, lists, exp_alive=None, exp_area=None):
    """replay `lists` into gb; pass_alive equals the restatement (and the expected values where given) point for
    point, the stored games are only read; returns (stones, alive, area)"""
    n = gb.board_size
    gb.replay(lists)
    h0, i0, l0 = gb.getHashCode(), gb.info(), gb.legal_mask()
    stones = gb.stones()
    alive, area = gb.pass_alive()
    assert alive.dtype == np.uint8 and area.dtype == np.uint8 and alive.shape == area.shape == (len(lists), n * n)
    for g in range(len(lists)):
        ea, er = B.benson(stones[g], n)
        np.testing.assert_array_equal(alive[g], ea, err_msg=f"alive of position {g}")
        np.testing.assert_array_equal(area[g], er, err_msg=f"area of position {g}")
    if exp_alive is not None:
        np.testing.assert_array_equal(alive, exp_alive)
        np.testing.assert_array_equal(area, exp_area)
    check_invariants(stones, alive, area)
    np.testing.assert_array_equal(gb.getHashCode(), h0)
    np.testing.assert_array_equal(gb.info(), i0)
    np.testing.assert_array_equal(gb.legal_mask(), l0)
    return stones, alive, area


def owner_passes_property(gb, alive, rng, plies=200):
    """the stored games: the colour with more pass-alive stones passes, the other plays uniformly random legal
    moves, for `plies` plies or until the game ends; every alive stone stays on the board at every ply"""
    n, G = gb.board_size, gb.num_games
    st0 = gb.stones()
    al = alive.astype(bool)
    owner = np.where((al & (st0 == 1)).sum(1) >= (al & (st0 == 2)).sum(1), 1, 2)
    moved = 0
    for _ in range(plies):
        term, info, legal = gb.terminated(), gb.info(), gb.legal_mask()[:, :-1]
        if term.all():
            break
        has = legal.any(1)
        pick = (rng.random(legal.shape) * legal).argmax(1)  # uniform among the legal moves
        opp = info[:, 1] != owner
        acts = np.where(opp & has, pick, n * n).astype(np.int32)
        acts[term] = -1  # no move for a finished game
        moved += int((opp & has & ~term).sum())
        assert gb.forward(acts)[acts >= 0].all()
        st = gb.stones()
        assert (st[al] == st0[al]).all(), "a pass-alive stone was captured"
    return moved


def expected_dead(stones, alive, area, dead_playout=None):
    dead = ((area == 1) & (stones == 2)) | ((area == 2) & (stones == 1))
    if dead_playout is not None:
        dead |= dead_playout.astype(bool) & ~alive.astype(bool)
    return dead.astype(np.uint8)


def run_final_status(gb, refs, stones, alive, area, K=4):
    """final_status(pass_alive=True) with and without counts against the rule restated, and its territory and
    score against the reference's getTrompTaylorScore with that dead set (refs: reference states, or None)"""
    from tests.test_ownership import ref_tt_territory

    counts = gb.ownership(K, seed=5)
    for c, k in ((None, None), (counts, K)):
        base = gb.final_status(c, k, 0.5)
        dead, terr, score = gb.final_status(c, k, 0.5, pass_alive=True)
        exp = expected_dead(stones, alive, area, base[0] if c is not None else None)
        np.testing.assert_array_equal(dead, exp)
        assert not (dead.astype(bool) & alive.astype(bool)).any()
        if refs is not None:
            for g, r in enumerate(refs):
                et, es = ref_tt_territory(r, dead[g])
                np.testing.assert_array_equal(terr[g], et, err_msg=f"territory of game {g}")
                assert score[g] == es, f"score of game {g}"
        # the default is today's call, unchanged
        again = gb.final_status(c, k, 0.5)
        for a, b in zip(base, again):
            np.testing.assert_array_equal(a, b)
    return counts


# ---- the restatement alone -----------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [9, 19])
def test_restatement_hand_built(n):
    for name, _, black, white, al, ar in all_hand_cases(n):
        s = np.zeros(n * n, np.uint8)
        s[black] = 1
        s[white] = 2
        a, r = B.benson(s, n)
        np.testing.assert_array_equal(a, al, err_msg=name)
        np.testing.assert_array_equal(r, ar, err_msg=name)


# ---- SIMT emulator -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    from tests import emu as E

    try:
        E.emu_lib()
    except Exception as e:  # no g++ / ucontext: the emulator is a convenience, not a requirement
        pytest.skip(f"SIMT emulator build unavailable: {e}")
    return E


@pytest.fixture(params=["ascending", "reverse", "random"])
def lane_order(request, emu):
    L = emu.emu_lib()
    L.simt_emu_set_order(["ascending", "reverse", "random"].index(request.param))
    yield request.param
    L.simt_emu_set_order(0)


_corpus = {}


def corpus(n, kind):
    """terminal ("end") or about 150-ply ("mid", 40 on 9x9) positions of the eye-avoiding random policy"""
    key = (n, kind)
    if key not in _corpus:
        _corpus[key] = corpus_chunk((n, 100 + n + (kind == "mid"), 8 if n == 19 else 12,
                                     None if kind == "end" else (150 if n == 19 else 40)))
    return _corpus[key]


@pytest.mark.parametrize("n", [9, 19])
def test_hand_built_positions(emu, lane_order, n):
    cases = all_hand_cases(n)
    gb = emu.emu_batch(len(cases), n)
    lists = [c[1] for c in cases]
    gb.replay(lists)
    st = gb.stones()
    for g, (name, _, black, white, _, _) in enumerate(cases):
        want = np.zeros(n * n, np.uint8)
        want[black] = 1
        want[white] = 2
        np.testing.assert_array_equal(st[g], want, err_msg=f"setup of {name}")
    run_equal_restatement(gb, lists, np.array([c[4] for c in cases]), np.array([c[5] for c in cases]))
    gb.close()


@pytest.mark.parametrize("n,kind", [(9, "end"), (19, "end"), (9, "mid"), (19, "mid")])
def test_random_policy_positions(emu, lane_order, n, kind):
    lists, stones, ea, er = corpus(n, kind)
    gb = emu.emu_batch(len(lists), n)
    st, alive, area = run_equal_restatement(gb, lists)
    np.testing.assert_array_equal(st, stones)
    np.testing.assert_array_equal(alive, ea)
    np.testing.assert_array_equal(area, er)
    if kind == "end":
        assert alive.sum() > 0 and (area > 0).sum() > 0  # not vacuous
    gb.close()


@pytest.mark.parametrize("n", [9, 19])
def test_golden_and_special_positions(emu, n):
    """tests/golden/positions_{9,19}.json, and the mix of tests/test_gather.py: an active ko, a handicap
    position, games ended by two passes, by superko (9x9) and by the ply cap (9x9), a mid-game position"""
    import json

    from tests.test_gather import make_sources
    from tests.test_handicap import need_ref

    here = os.path.dirname(os.path.abspath(__file__))
    games = {e["game_id"]: e for e in json.load(open(os.path.join(here, "golden", f"playouts_{n}.json")))["games"]
             if "moves" in e}
    pos = [p for p in json.load(open(os.path.join(here, "golden", f"positions_{n}.json")))["positions"]
           if p["game_id"] in games and p["after_ply"] <= games[p["game_id"]]["plies"]]
    lists = [games[p["game_id"]]["moves"][: p["after_ply"]] for p in pos]
    gb = emu.emu_batch(len(lists), n)
    st, _, _ = run_equal_restatement(gb, lists)
    np.testing.assert_array_equal(st, np.array([p["stones"] for p in pos], np.uint8))
    gb.close()
    need_ref(n)
    src, refs = make_sources(emu.emu_batch, n, np.random.default_rng(n))
    stones = src.stones()
    h0, i0 = src.getHashCode(), src.info()
    alive, area = src.pass_alive()
    for g in range(src.num_games):
        ea, er = B.benson(stones[g], n)
        np.testing.assert_array_equal(alive[g], ea)
        np.testing.assert_array_equal(area[g], er)
    np.testing.assert_array_equal(src.getHashCode(), h0)
    np.testing.assert_array_equal(src.info(), i0)
    info = np.array([r.info() for r in refs])
    assert info[:, 10].any() and info[:, 9].any()  # two passes, and ended games
    if n == 9:
        assert info[:, 11].any()  # superko
    src.close()


@pytest.mark.parametrize("n", [9, 19])
def test_owner_passes_alive_stones_survive(emu, n):
    lists, stones, ea, _ = corpus(n, "end")
    keep = [g for g in range(len(lists)) if ea[g].any()]
    lists = [lists[g] for g in keep]
    for mv in lists:  # drop the closing passes, so that the game goes on from the same stones
        while mv and mv[-1] == n * n:
            mv.pop()
    gb = emu.emu_batch(len(lists), n)
    gb.replay(lists)
    alive, _ = gb.pass_alive()
    assert alive.any()
    moved = owner_passes_property(gb, alive, np.random.default_rng(7), plies=200 if n == 9 else 60)
    assert moved > 0
    gb.close()


def test_final_status_pass_alive(emu, lane_order):
    from tests.test_handicap import need_ref

    n = 9
    lists, _, _, _ = corpus(n, "end")
    cases = all_hand_cases(n)
    lists = lists + [c[1] for c in cases[::5]]
    gb = emu.emu_batch(len(lists), n)
    stones, alive, area = run_equal_restatement(gb, lists)
    refs = None
    if oracles.have_ref(n):
        refs = []
        for mv in lists:
            r = oracles.Ref(n)
            for a in mv:
                r.forward(a)
            refs.append(r)
    run_final_status(gb, refs, stones, alive, area)
    assert ((area == 1) & (stones == 2)).any() or ((area == 2) & (stones == 1)).any()  # certain dead stones met
    gb.close()
    need_ref(n)  # report the reference scorer's absence (the rest above ran without it)


def test_null_outputs_and_arguments(emu):
    L = emu.emu_lib()
    n = 9
    lists, _, _, _ = corpus(n, "end")
    gb = emu.emu_batch(len(lists), n)
    gb.replay(lists)
    alive, area = gb.pass_alive()
    G, P = len(lists), n * n
    for want in ((1, 0), (0, 1), (1, 1)):
        for fn in (L.elfb200_pass_alive, L.elfb200_pass_alive_dev):  # host buffers stand for device memory here
            bufs = [np.full((G, P), 9, np.uint8) for _ in range(2)]
            n0 = gb.launch_count()
            assert fn(gb._ctx, *[b.ctypes.data if w else None for b, w in zip(bufs, want)]) == 0
            assert gb.launch_count() == n0 + 1
            for b, w, exp in zip(bufs, want, (alive, area)):
                np.testing.assert_array_equal(b, exp if w else np.full_like(b, 9))
    n0 = gb.launch_count()
    assert L.elfb200_pass_alive(gb._ctx, None, None) == 0 and L.elfb200_pass_alive_dev(gb._ctx, None, None) == 0
    assert gb.launch_count() == n0  # nothing asked, nothing launched
    buf = np.zeros((G, P), np.uint8)
    assert L.elfb200_pass_alive(None, buf.ctypes.data, None) == ERR_ARG
    assert L.elfb200_pass_alive_dev(None, buf.ctypes.data, None) == ERR_ARG
    assert L.elfb200_final_status_pass_alive(None, None, 1, 0.5, buf.ctypes.data, None, None) == ERR_ARG
    c = np.zeros((G, 2, P), np.int32)
    assert L.elfb200_final_status_pass_alive(gb._ctx, c.ctypes.data, 0, 0.5, None, None, None) == ERR_ARG
    assert L.elfb200_final_status_pass_alive(gb._ctx, None, 1, float("nan"), None, None, None) == ERR_ARG
    with pytest.raises(ValueError):
        gb.pass_alive(out=(np.zeros((G, P), np.uint8), None))  # not a CUDA tensor
    gb.close()
    e = emu.emu_batch(2, n)  # the empty board: nothing
    a, r = e.pass_alive()
    assert not a.any() and not r.any()
    e.close()


def test_gtp_final_status_list_pass_alive(emu):
    """the finished 9x9 game of tests/test_ownership.py: black's and white's two-eyed groups are pass-alive, the
    white stone inside black's eye region is certainly dead"""
    from tests.test_handicap import make_console, need_ref
    from tests.test_ownership import endgame_9, run_gtp_final_status

    need_ref(9)
    g, console = make_console(emu, 9)
    assert console.final_status_pass_alive is False
    console.final_status_playouts = 16
    console.final_status_pass_alive = True
    run_gtp_final_status(g, console)
    black, white, dead = endgame_9()
    alive, area = g._final.pass_alive()
    assert alive[0][black + [a for a in white if a not in dead]].all() and area[0][dead].tolist() == [1]
    dg, ag = g.final_status(playouts=16, pass_alive=True)
    assert dg == [dead]


_ASAN_CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests/simt_emu")
import build
from elf_b200 import lib as _l
from tests import emu as E
from tests import test_pass_alive as TP
E._lib = _l.load_library(build.build(asan=True))
for n in (19, 9):
    cases = TP.all_hand_cases(n)
    lists = [c[1] for c in cases[::3]] + TP.corpus(n, "end")[0][:4]
    gb = E.emu_batch(len(lists), n)
    st, alive, area = TP.run_equal_restatement(gb, lists)
    out = np.zeros((2, len(lists), n * n), np.uint8)
    _l.check(E._lib, E._lib.elfb200_pass_alive_dev(gb._ctx, out[0].ctypes.data, out[1].ctypes.data))
    assert (out[0] == alive).all() and (out[1] == area).all()
    d, t, s = gb.final_status(pass_alive=True)
    assert (d == TP.expected_dead(st, alive, area)).all()
    gb.close()
print("ASAN PASS_ALIVE CLEAN")
"""


def test_pass_alive_clean_under_address_sanitizer(emu):
    """the kernels on hand-built and random-policy positions on the emulator build under AddressSanitizer"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    try:
        asan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        pytest.skip(f"no gcc: {e}")
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("libasan is not installed")
    env = dict(os.environ, LD_PRELOAD=os.path.realpath(asan), ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0")
    r = subprocess.run([sys.executable, "-c", _ASAN_CHILD, root], env=env, capture_output=True, text=True, timeout=850)
    assert r.returncode == 0 and "ASAN PASS_ALIVE CLEAN" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]
