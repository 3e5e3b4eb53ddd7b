"""Ladders and self-ataris (elfb200_tactics / elfb200_tactics_dev, k_tactics, GoBatch.tactics) against the compiled
reference's checkLadder, checkLadderUseSearch and isSelfAtari (board.cc:242-524), triple for triple: every point,
both colours, the ladder depth, the self-atari size and the number of search calls.

CPU: the kernel runs on the SIMT emulator build of the kernel sources (tests/simt_emu) under every lane order.
tests/test_zz_gpu_tactics.py runs the checks on the whole ladder suite and full batches on an H100."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import tactics_ref as T
from tests.test_handicap import need_ref

pytestmark = pytest.mark.timeout(900)

ERR_ARG = -1  # ELFB200_ERR_ARG (include/elfb200.h)
N = 19
P = N * N


def A(x, y):
    return x * N + y


def setup(black, white, to_move=1):
    """a move list that places the stones (black and white alternate, a pass where one colour has none left) and
    leaves `to_move` to play; a list that would need two passes in a row at the end ends the game instead, which
    the tactics do not look at"""
    b, w = list(black), list(white)
    mv = []
    while b or w:
        mv.append(b.pop(0) if b else P)
        mv.append(w.pop(0) if w else P)
    if mv and mv[-1] == P:
        mv.pop()  # white to move
    if (len(mv) % 2 == 0) != (to_move == 1):
        mv.append(P)
    return mv


# A white stone at D4 (3, 3) in atari from black (2, 3), (3, 2), (4, 3); black (2, 4) joins (2, 3) in a group of four
# liberties.  White's escape at (3, 4) has two empty neighbours, the own group in atari and one enemy group with
# >= 3 liberties: checkLadder searches.  Black blocks (3, 5) (three empty neighbours: must_block), white flees to
# (4, 4), and so on diagonally towards (18, 18), where white is caught at the edge.
LADDER_B = [A(2, 3), A(3, 2), A(4, 3), A(2, 4)]
LADDER_W = [A(3, 3)]
ESCAPE = A(3, 4)


def hand_built():
    """(name, move list, what the reference gives at the escape for white: (depth, calls) or None to check only)"""
    # a ko shape at (10, 10) / (11, 10): white's last move at (10, 10) takes black (11, 10), which black may not
    # retake at once
    ko_b, ko_w = [A(9, 10), A(10, 9), A(10, 11), A(11, 10)], [A(11, 9), A(11, 11), A(12, 10)]
    return [
        ("ladder to the edge, black to move", setup(LADDER_B, LADDER_W, 1), (57, 57)),
        ("ladder to the edge, white to move", setup(LADDER_B, LADDER_W, 2), (57, 57)),
        # a white stone on the diagonal: white connects to it and has three liberties
        ("ladder breaker", setup(LADDER_B, LADDER_W + [A(12, 12)]), (0, 33)),
        # white (5, 3) leaves black (4, 3) one liberty once white flees to (4, 4) with two: not a ladder, found by
        # the second call
        ("flee puts a capturer stone in atari", setup(LADDER_B, LADDER_W + [A(5, 3)]), (0, 2)),
        # black (5, 6) takes a free point from both escapes at one capturer node: escape[0] is read on a copy and
        # fails, escape[1] on the board catches white (10 calls for a depth of 7)
        ("branching node", setup(LADDER_B + [A(5, 6)], LADDER_W), (7, 10)),
        # the same ladder runs into an active simple ko (black, the colour to move, may not retake): its path
        # reaches the ko shape after 25 calls and white gets out there
        ("ladder through a simple ko", setup(LADDER_B + ko_b, LADDER_W + ko_w, 2) + [A(10, 10)], (0, 25)),
    ]


def run_equal_reference(make_batch, n, lists, order=None, seen=None):
    """GoBatch.tactics of the positions `lists` equals the reference for every triple; returns the values"""
    need_ref(n)
    gb = make_batch(len(lists), n)
    gb.replay(lists)
    h0, i0, l0 = gb.getHashCode(), gb.info(), gb.legal_mask()
    lad, sa, calls = gb.tactics(trace=True)
    assert lad.dtype == np.int16 and sa.dtype == np.int16 and calls.dtype == np.int32
    assert lad.shape == sa.shape == calls.shape == (len(lists), 2, n * n)
    for g, moves in enumerate(lists):
        r = T.ref_of(n, moves)
        assert int(h0[g]) == r.hash()
        for name, got, want in zip(("ladder", "self_atari", "calls"), (lad[g], sa[g], calls[g]), T.ref_tactics(r)):
            bad = np.argwhere(got != want)
            assert len(bad) == 0, (f"{name} of position {g}: (colour, action, got, want) "
                                   f"{[(int(c), int(a), int(got[c, a]), int(want[c, a])) for c, a in bad[:5]]}")
    # the stored games are only read
    np.testing.assert_array_equal(gb.getHashCode(), h0)
    np.testing.assert_array_equal(gb.info(), i0)
    np.testing.assert_array_equal(gb.legal_mask(), l0)
    assert (lad >= 0).all()  # no search reached the path cap
    if seen is not None:  # the same values under every lane order
        key = (n, len(lists))
        if key in seen:
            for a, b in zip((lad, sa, calls), seen[key]):
                np.testing.assert_array_equal(a, b, err_msg=f"lane order {order}")
        seen[key] = (lad, sa, calls)
    gb.close()
    return lad, sa, calls


_suite = {}


def suite_subset():
    """ladder-suite positions: every one with a ladder in the first 60 records until they hold >= 200 ladders,
    plus every 40th position of the whole suite"""
    if not _suite:
        lists = T.ladder_suite_lists()
        picked, ladders = [], 0
        for i, moves in enumerate(lists[:6500]):
            if ladders >= 220:
                break
            lad = T.ref_tactics(T.ref_of(N, moves), skip_open=True)[0]
            if (lad > 0).any():
                picked.append(i)
                ladders += int((lad > 0).sum())
        picked = sorted(set(picked) | set(range(0, len(lists), 40)))
        _suite["lists"] = [lists[i] for i in picked]
    return _suite["lists"]


# ---- SIMT emulator -----------------------------------------------------------------------------------------
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


_seen = {}


def test_ladder_suite_positions_equal_reference(emu, lane_order):
    need_ref(N)
    lists = suite_subset()
    lad, _, calls = run_equal_reference(emu.emu_batch, N, lists, lane_order, _seen)
    assert (lad > 0).sum() >= 200
    assert ((calls > 0) & (lad == 0)).any()  # searches that fail as well


@pytest.mark.parametrize("n,plies", [(9, (10, 30, 50, 70)), (19, (40, 120, 220))])
def test_random_positions_equal_reference(emu, lane_order, n, plies):
    need_ref(n)
    rng = np.random.default_rng(n)
    lists = [T.random_game(n, rng, t) for t in plies for _ in range(5)]
    _, sa, _ = run_equal_reference(emu.emu_batch, n, lists, lane_order, _seen)
    assert (sa > 0).any()


def test_hand_built_positions_equal_reference(emu):
    need_ref(N)
    cases = hand_built()
    lists = [m for _, m, _ in cases]
    lad, sa, calls = run_equal_reference(emu.emu_batch, N, lists)
    for g, (name, moves, want) in enumerate(cases):
        if want is not None:
            assert (int(lad[g, 1, ESCAPE]), int(calls[g, 1, ESCAPE])) == want, name
    info = np.array([T.ref_of(N, m).info() for m in lists])
    assert list(info[:2, 1]) == [1, 2]  # the ladder is read for white whoever is to move
    g = len(cases) - 1
    assert info[g, 1] == 1 and info[g, 6] == A(11, 10) and info[g, 7] == 1  # an active ko for black, to move
    assert sa[g, 0, A(11, 10)] == 0 and sa[g, 1, A(11, 10)] == 0  # the ko point: illegal for black, not for white


def test_call_budget():
    """checkLadderUseSearch stops branching once 1024 calls are made (MAX_LADDER_SEARCH, board.cc:298).  No position
    that reaches the budget has been found, so that branch is not claimed as tested: the ladder suite needs at most
    77 calls, and a random search over a few extra stones around the hand-built ladder found at most 251.  This
    test records it with the branching case."""
    need_ref(N)
    r = T.ref_of(N, setup(LADDER_B + [A(5, 6)], LADDER_W))
    assert T.ref_tactics(r)[2].max() < 1024


def test_null_outputs_skip_work(emu):
    need_ref(N)
    L = emu.emu_lib()
    lists = [c[1] for c in hand_built()]
    gb = emu.emu_batch(len(lists), N)
    gb.replay(lists)
    lad, sa, calls = gb.tactics(trace=True)
    G = len(lists)
    for want in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0)):
        bufs = [np.full((G, 2, P), -5, dt) for dt in (np.int16, np.int16, np.int32)]
        ptrs = [b.ctypes.data if w else None for b, w in zip(bufs, want)]
        n0 = gb.launch_count()
        assert L.elfb200_tactics(gb._ctx, *ptrs) == 0
        assert gb.launch_count() == n0 + 1
        for b, w, exp in zip(bufs, want, (lad, sa, calls)):
            if w:
                np.testing.assert_array_equal(b, exp)
            else:
                assert (b == -5).all()
    # the device form, with host buffers standing for device memory on the emulator
    for want in ((1, 1), (1, 0), (0, 1)):
        bufs = [np.full((G, 2, P), -5, np.int16) for _ in range(2)]
        assert L.elfb200_tactics_dev(gb._ctx, *[b.ctypes.data if w else None for b, w in zip(bufs, want)]) == 0
        for b, w, exp in zip(bufs, want, (lad, sa)):
            np.testing.assert_array_equal(b, exp if w else np.full_like(b, -5))
    n0 = gb.launch_count()
    assert L.elfb200_tactics(gb._ctx, None, None, None) == 0 and L.elfb200_tactics_dev(gb._ctx, None, None) == 0
    assert gb.launch_count() == n0  # nothing asked, nothing launched
    gb.close()


def test_arguments(emu):
    L = emu.emu_lib()
    gb = emu.emu_batch(2, 9)
    buf = np.zeros(2 * 2 * 81 + 1, np.int16)
    assert L.elfb200_tactics(None, buf.ctypes.data, None, None) == ERR_ARG
    assert L.elfb200_tactics_dev(None, buf.ctypes.data, None) == ERR_ARG
    assert L.elfb200_tactics_dev(gb._ctx, buf.ctypes.data + 1, None) == ERR_ARG
    assert L.elfb200_tactics_dev(gb._ctx, None, buf.ctypes.data + 1) == ERR_ARG
    assert b"aligned" in L.elfb200_last_error()
    with pytest.raises(ValueError):
        gb.tactics(out=(np.zeros((2, 2, 81), np.int16), None))  # not a CUDA tensor
    lad, sa = gb.tactics()  # the empty board: nothing to read
    assert not lad.any() and not sa.any()
    gb.close()


_ASAN_CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests/simt_emu")
import build
from elf_b200 import lib as _l
from tests import emu as E
from tests import test_tactics as TT
E._lib = _l.load_library(build.build(asan=True))
lists = [c[1] for c in TT.hand_built()] + TT.T.ladder_suite_lists(limit=2)[150:170]
for n, G in ((19, len(lists)), (9, 7)):
    gb = E.emu_batch(G, n)
    rng = np.random.default_rng(n)
    gb.replay(lists if n == 19 else [[int(a) for a in rng.integers(0, n * n + 1, int(rng.integers(0, 2 * n * n)))]
                                     for _ in range(G)])
    lad, sa, calls = gb.tactics(trace=True)
    out = np.zeros((2, G, 2, n * n), np.int16)
    _l.check(E._lib, E._lib.elfb200_tactics_dev(gb._ctx, out[0].ctypes.data, out[1].ctypes.data))
    assert (out[0] == lad).all() and (out[1] == sa).all()
    gb.close()
print("ASAN TACTICS CLEAN")
"""


def test_tactics_clean_under_address_sanitizer(emu):
    """the kernel on hand-built, ladder-suite and random positions on the emulator build under AddressSanitizer
    (every device buffer is a heap allocation there, so any read or write outside one is reported)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    need_ref(N)
    try:
        asan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        pytest.skip(f"no gcc: {e}")
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("libasan is not installed")
    env = dict(os.environ, LD_PRELOAD=os.path.realpath(asan), ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0")
    r = subprocess.run([sys.executable, "-c", _ASAN_CHILD, root], env=env, capture_output=True, text=True, timeout=850)
    assert r.returncode == 0 and "ASAN TACTICS CLEAN" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]
