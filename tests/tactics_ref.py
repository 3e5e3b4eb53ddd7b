"""The reference side of the ladder and self-atari checks (elfb200_tactics, k_tactics): the compiled reference's
TryPlay, checkLadder, isSelfAtari, Play and checkLadderUseSearch (board.cc:242-524, 788-827), bound by their C++
symbol names as tests/test_ownership.py binds getTrompTaylorScore, and the positions both sides are compared on.
Shared by tests/test_tactics.py (SIMT emulator) and tests/test_zz_gpu_tactics.py (H100)."""
import ctypes
import gzip
import json
import os

import numpy as np

from elf_b200 import sgf
from tests import oracles
from tests.test_gather import ref_clone

LADDER_SUITE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ladder_suite.json.gz")

_SYMBOLS = {  # name -> (mangled name, restype, argtypes)
    "TryPlay": ("_Z7TryPlayPK5BoardiihP8GroupId4", ctypes.c_bool,
                [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_ubyte, ctypes.c_void_p]),
    "checkLadder": ("_Z11checkLadderPK5BoardPK8GroupId4h", ctypes.c_int,
                    [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_ubyte]),
    "isSelfAtari": ("_Z11isSelfAtariPK5BoardPK8GroupId4thPi", ctypes.c_bool,
                    [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_ushort, ctypes.c_ubyte, ctypes.c_void_p]),
    "Play": ("_Z4PlayP5BoardPK8GroupId4", ctypes.c_bool, [ctypes.c_void_p, ctypes.c_void_p]),
    "checkLadderUseSearch": ("_Z20checkLadderUseSearchP5BoardhPii", ctypes.c_int,
                             [ctypes.c_void_p, ctypes.c_ubyte, ctypes.c_void_p, ctypes.c_int]),
}


class GroupId4(ctypes.Structure):  # board.h:78-85
    _fields_ = [("c", ctypes.c_ushort), ("player", ctypes.c_ubyte), ("ids", ctypes.c_short * 4),
                ("colors", ctypes.c_ubyte * 4), ("group_liberties", ctypes.c_short * 4), ("liberty", ctypes.c_short)]


_fns = {}


def ref_fns(n):
    if n not in _fns:
        L = oracles.load_ref(n)
        f = {}
        for name, (sym, res, args) in _SYMBOLS.items():
            fn = getattr(L, sym)
            fn.restype, fn.argtypes = res, args
            f[name] = fn
        _fns[n] = f
    return _fns[n]


def ladder_preconditions(ids, player):
    """checkLadder's cheap test before its search (board.cc:478-511), quirks included: a second enemy or own
    group clears the flag whatever the first one was"""
    if ids.liberty != 2:
        return False
    n_enemy = n_self = 0
    enemy3 = atari1 = False
    for i in range(4):
        if ids.ids[i] & 0xFF == 0:  # `unsigned char id = ids->ids[i]`
            continue
        if ids.colors[i] == 3 - player:
            enemy3 = False if n_enemy >= 1 else (enemy3 or ids.group_liberties[i] >= 3)
            n_enemy += 1
        else:
            atari1 = False if n_self >= 1 else (atari1 or ids.group_liberties[i] == 1)
            n_self += 1
    return enemy3 and atari1


def ref_tactics(r, skip_open=False):
    """(ladder int16[2][P], self_atari int16[2][P], calls int32[2][P]) of reference state r, as elfb200_tactics
    defines them.  calls is num_call of checkLadderUseSearch on a copy of r after Play, as checkLadder runs it.
    skip_open=True leaves out the points where the answer is 0 by the definition alone: stones, and empty points
    with three or four empty neighbours (TryPlay's ids.liberty >= 3 fails checkLadder's first test and
    isSelfAtari's first test)."""
    n, P = r.n, r.n * r.n
    f = ref_fns(n)
    lad = np.zeros((2, P), np.int16)
    sa = np.zeros((2, P), np.int16)
    calls = np.zeros((2, P), np.int32)
    points = range(P)
    if skip_open:
        st = r.stones().reshape(n, n)  # [x][y]
        e = np.pad(st == 0, 1)
        ne = e[:-2, 1:-1].astype(int) + e[2:, 1:-1] + e[1:-1, :-2] + e[1:-1, 2:]
        points = np.flatnonzero(((st == 0) & (ne <= 2)).reshape(-1))
    ids = GroupId4()
    k = ctypes.c_int(0)
    for a in points:
        a = int(a)
        for ci, player in enumerate((1, 2)):
            if not f["TryPlay"](r.p, a // n, a % n, player, ctypes.byref(ids)):
                continue
            lad[ci, a] = f["checkLadder"](r.p, ctypes.byref(ids), player)
            k.value = 0
            if f["isSelfAtari"](r.p, ctypes.byref(ids), ids.c, player, ctypes.byref(k)):
                sa[ci, a] = k.value
            if ladder_preconditions(ids, player):
                b = ref_clone(r)
                f["Play"](b.p, ctypes.byref(ids))
                k.value = 0
                d = f["checkLadderUseSearch"](b.p, player, ctypes.byref(k), 1)
                assert d == lad[ci, a], "checkLadder and its search disagree"
                calls[ci, a] = k.value
    return lad, sa, calls


def ladder_suite_lists(limit=None):
    """every position of the ladder_suite records (the reference's ladder_suite/ CGOS games): the move list of
    each prefix of each record, in record order"""
    lists = []
    for rec in json.load(gzip.open(LADDER_SUITE, "rt"))["records"][:limit]:
        moves = []
        for m in sgf.Sgf.loads(rec["sgf"]):
            if m.action < 0:
                break
            moves.append(int(m.action))
            lists.append(list(moves))
    return lists


def ref_of(n, moves):
    r = oracles.Ref(n)
    for a in moves:
        assert r.forward(a)
    return r


def random_game(n, rng, plies):
    """up to `plies` uniform legal moves on a fresh reference state (a pass when none is legal); the moves"""
    r = oracles.Ref(n)
    moves = []
    for _ in range(plies):
        if r.terminated():
            break
        cand = np.flatnonzero(r.legal())
        a = int(rng.choice(cand)) if len(cand) else n * n
        assert r.forward(a)
        moves.append(a)
    return moves


def ref_chunk(args):
    """reference values of a chunk of move lists: stacked (ladder, self_atari, calls)"""
    n, lists, skip_open = args
    out = [ref_tactics(ref_of(n, m), skip_open) for m in lists]
    return tuple(np.stack([o[j] for o in out]) for j in range(3))
