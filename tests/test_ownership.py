"""Monte-Carlo ownership and dead stones (elfb200_ownership / elfb200_final_status, k_ownership / k_final_status,
GoBatch.ownership / final_status, OnlineGame.final_status, GTP final_status_list) against the compiled reference.

The reference side: every playout is GoState::forward on a copy (ref_clone) of the source state, with the policy of
include/elfb200_playout_policy.h, and every territory map and score is the reference's getTrompTaylorScore(board,
group_stats, territory) (board.cc:1954-2071), bound by its C++ symbol name as tests/test_handicap.py binds
PlaceHandicap.

CPU: the kernels run on the SIMT emulator build of the kernel sources (tests/simt_emu) under every lane order.
tests/test_zz_gpu_ownership.py runs the checks at full batch size on an H100."""
import ctypes

import numpy as np
import pytest

from tests import oracles
from tests.test_gather import make_sources, ref_clone
from tests.test_handicap import make_console, need_ref

pytestmark = pytest.mark.timeout(900)

ERR_ARG = -1  # ELFB200_ERR_ARG (include/elfb200.h)
M_INVALID = 3  # common.h:47
S_DEAD = 8  # board.h:425
MAX_GROUP = 173  # board.h:90
_TT = "_Z19getTrompTaylorScorePK5BoardPKhPh"  # getTrompTaylorScore(const Board*, const Stone*, Stone*)


# ---- the reference side ------------------------------------------------------------------------------------
class _Info(ctypes.Structure):  # Info, board.h:57-67
    _fields_ = [("color", ctypes.c_ubyte), ("id", ctypes.c_ubyte), ("next", ctypes.c_ushort),
                ("last_placed", ctypes.c_ushort)]


class _Group(ctypes.Structure):  # Group, board.h:69-74
    _fields_ = [("color", ctypes.c_ubyte), ("start", ctypes.c_ushort), ("stones", ctypes.c_short),
                ("liberties", ctypes.c_short)]


_heads = {}


def _board_head(n):
    """the leading fields of the reference Board (board.h:95-125) up to _last_move2; the shim's state object is
    a GoState whose first member is its Board (see tests/test_handicap.py), so the state pointer addresses it"""
    if n not in _heads:
        E = n + 2

        class Head(ctypes.Structure):
            _fields_ = [("infos", _Info * (E * E)), ("bits", ctypes.c_ubyte * (E * E // 4 + 1)),
                        ("hash", ctypes.c_uint64), ("groups", _Group * MAX_GROUP), ("num_groups", ctypes.c_short),
                        ("b_cap", ctypes.c_short), ("w_cap", ctypes.c_short), ("rollout_passes", ctypes.c_short),
                        ("last_move", ctypes.c_ushort), ("last_move2", ctypes.c_ushort)]

        _heads[n] = Head
    return _heads[n]


def coord(a, n):
    """OFFSETXY(x, y) of action a = x*N + y (board.h:183-190)"""
    return (a % n + 1) * (n + 2) + a // n + 1


def board_of(r):
    """the reference Board of state r, checked against what the shim reports"""
    h = _board_head(r.n).from_address(r.p)
    i = r.info()
    assert h.hash == r.hash() and h.b_cap == i[2] and h.w_cap == i[3], "Board layout does not match the reference"
    for fld, act in (("last_move", i[4]), ("last_move2", i[5])):
        want = 0 if act == r.n * r.n else (M_INVALID if act < 0 else coord(int(act), r.n))  # M_PASS = 0
        assert getattr(h, fld) == want, "Board layout does not match the reference"
    return h


def _tt_fn(n):
    f = getattr(oracles.load_ref(n), _TT)
    f.restype, f.argtypes = ctypes.c_float, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return f


def ref_tt_territory(r, dead=None):
    """getTrompTaylorScore with S_DEAD in group_stats on the group id of every stone with dead[a] != 0:
    (territory uint8[N*N] by action, score)"""
    n = r.n
    h = board_of(r)
    stats = (ctypes.c_ubyte * MAX_GROUP)()
    if dead is not None:
        for a in np.flatnonzero(dead):
            stats[h.infos[coord(int(a), n)].id] = S_DEAD
    terr = np.zeros(n * n, np.uint8)
    score = _tt_fn(n)(r.p, ctypes.addressof(stats) if dead is not None else None, terr.ctypes.data)
    return terr, int(score)


def ref_groups(r):
    """group id of every stone by action (0 on empty points), from the reference's own group table"""
    h = board_of(r)
    return np.array([h.infos[coord(a, r.n)].id for a in range(r.n * r.n)], np.int32)


_M = (1 << 64) - 1


def _splitmix(x):
    x = (x + 0x9E3779B97F4A7C15) & _M
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M
    return x ^ (x >> 31)


def pp_pick(seed, gid, ply, n):  # include/elfb200_playout_policy.h
    r = _splitmix(seed ^ ((gid * 0x9E3779B97F4A7C15) & _M) ^ ply)
    return ((r >> 32) * n) >> 32


def ref_playout_from(r, seed, pid, max_plies):
    """one playout of the policy from a copy of reference state r with draw id pid: (plies, final hash,
    getTrompTaylorScore territory of the final position, score).  A state ended by two passes is played on with
    its last-move window cleared (isTwoPass reads Board::_last_move / _last_move2)."""
    n, P = r.n, r.n * r.n
    c = ref_clone(r)
    if c.info()[10]:
        h = board_of(c)
        h.last_move = h.last_move2 = M_INVALID
    t = 0
    while not c.terminated() and t < max_plies:
        i = c.info()
        cand = np.flatnonzero(c.legal() & (c.true_eyes(int(i[1])) ^ 1))
        a = P if len(cand) == 0 else int(cand[pp_pick(seed, pid, int(i[0]), len(cand))])
        assert c.forward(a)
        t += 1
    terr, score = ref_tt_territory(c)
    return t, c.hash(), terr, score


def dead_rule(r, counts, K, threshold):
    """the dead rule restated over the reference's groups: a group of colour c is dead iff the sum over its stones
    of (own area count - opponent area count) < -threshold * K * |S|"""
    st, ids = r.stones(), ref_groups(r)
    dead = np.zeros(r.n * r.n, np.uint8)
    for gid in np.unique(ids[st > 0]):
        S = np.flatnonzero((ids == gid) & (st > 0))
        c = int(st[S[0]])
        own = int(counts[0, S].astype(np.int64).sum() - counts[1, S].astype(np.int64).sum())
        own = own if c == 1 else -own
        if float(own) < -threshold * K * len(S):
            dead[S] = 1
    return dead


# ---- corpus ------------------------------------------------------------------------------------------------
def superko_fixture(n, seed, K):
    """(slot, moves to replay, T) of a playout from the empty board that ends by positional superko at ply T
    against a hash first recorded at ply t0: its first s moves with t0 < s < T, for slot g = id / K (an id that K
    divides).  The first playout from there has draw id g*K = the game id: it replays the rest and ends by the same
    superko, which it finds only in the source record."""
    for gid in range(0, 20000, K):
        t, _, _, moves, hashes, _ = oracles.oracle_playout(n, seed, gid, trace=True)
        pre = [0] + [int(h) for h in hashes[: t - 1]]  # pre-move hashes; the record keeps those of stones
        final = int(hashes[t - 1])
        rec = [i for i in range(t - 1) if pre[i] == final and moves[i] != n * n]
        if t < 2 * n * n and moves[t - 1] != n * n and rec:
            t0 = rec[0]
            s = t0 + 1 + (t - 1 - t0) // 2
            assert t0 < s < t
            return gid // K, [int(a) for a in moves[:s]], t
    raise AssertionError("no playout ends by superko")


def build_corpus(make_batch, n, K, seed, rng):
    """make_sources' mix (fresh, active ko, handicap, two passes, mid-game; on 9x9 also superko and the ply cap)
    plus random positions of varied length and the superko fixture at slot g = its game id"""
    src, srefs = make_sources(make_batch, n, rng)
    gid, fixture, T = superko_fixture(n, seed, K)
    G = max(src.num_games + 4, gid + 1)
    gb = make_batch(G, n)
    refs = [None] * G
    lists = [None] * G
    for g in range(G):
        if g == gid:
            lists[g] = fixture
        elif src.num_games <= g < src.num_games + 4:
            r = oracles.Ref(n)
            lists[g] = []
            for _ in range(int(rng.integers(5, n * n))):
                if r.terminated():
                    break
                cand = np.flatnonzero(r.legal())
                a = int(rng.choice(cand)) if len(cand) else n * n
                r.forward(a)
                lists[g].append(a)
    # the games copied from the mix keep their state; every slot left over holds the full superko game, which
    # has ended and plays no move
    t, _, _, moves, _, _ = oracles.oracle_playout(n, seed, gid * K, trace=True)
    filler = [int(a) for a in moves[:t]]
    for g in range(G):
        if lists[g] is None and g >= src.num_games:
            lists[g] = filler
    gb.replay([lst if lst is not None else [] for lst in lists])
    idx = np.array([g if g < src.num_games and lists[g] is None else -1 for g in range(G)], np.int32)
    gb.gather(src, idx)
    for g in range(G):
        if idx[g] >= 0:
            refs[g] = ref_clone(srefs[g])
        else:
            refs[g] = oracles.Ref(n)
            for a in lists[g]:
                refs[g].forward(a)
    np.testing.assert_array_equal(gb.getHashCode(), [r.hash() for r in refs])
    return gb, refs, gid, T - len(fixture)


# ---- checks ------------------------------------------------------------------------------------------------
_counts_seen = {}


def run_ownership_equals_reference(make_batch, n, K, seed, order):
    rng = np.random.default_rng(3 * n)
    gb, refs, gid, rest = build_corpus(make_batch, n, K, seed, rng)
    G, P, maxp = gb.num_games, n * n, 2 * n * n
    h0 = gb.getHashCode()
    counts, fh, plies = gb.ownership(K, seed=seed, trace=True)
    assert counts.shape == (G, 2, P) and fh.shape == (G, K) and plies.shape == (G, K)
    np.testing.assert_array_equal(gb.getHashCode(), h0)  # the stored games are only read
    for g in range(G):
        exp = np.zeros((2, P), np.int64)
        for k in range(K):
            t, h, terr, _ = ref_playout_from(refs[g], seed, g * K + k, maxp)
            assert (int(plies[g, k]), int(fh[g, k])) == (t, h), f"playout ({g}, {k})"
            exp[0] += terr == 1
            exp[1] += terr == 2
        np.testing.assert_array_equal(counts[g], exp, err_msg=f"counts of game {g}")
    # the superko fixture plays exactly the rest of its game and ends by the same superko
    assert plies[gid, 0] == rest and gb.info()[gid, 9] == 0
    # games ended by superko or the ply cap play no move; one ended by two passes plays on
    info = np.array([r.info() for r in refs])
    for g in range(G):
        if info[g, 9] and not info[g, 10]:
            assert (plies[g] == 0).all()
        if info[g, 10]:
            assert (plies[g] > 0).all()
    key = (n, K, seed)
    if key in _counts_seen:  # the same counts under every lane order
        np.testing.assert_array_equal(counts, _counts_seen[key], err_msg=f"lane order {order}")
    _counts_seen[key] = counts
    # max_plies bounds the moves of every playout
    _, _, p2 = gb.ownership(K, seed=seed, max_plies=3, trace=True)
    assert (p2 <= 3).all()
    return gb, refs, counts, K


def run_final_status_equals_reference(gb, refs, counts, K):
    n = gb.board_size
    seen = set()
    for thr in np.linspace(-1.0, 1.0, 9):
        dead, terr, score = gb.final_status(counts, K, float(thr))
        for g, r in enumerate(refs):
            exp = dead_rule(r, counts[g], K, float(thr))
            np.testing.assert_array_equal(dead[g], exp, err_msg=f"dead stones of game {g} at threshold {thr}")
            et, es = ref_tt_territory(r, exp)
            np.testing.assert_array_equal(terr[g], et, err_msg=f"territory of game {g} at threshold {thr}")
            assert score[g] == es
            seen.add((g, dead[g].tobytes()))
    assert len(seen) > len(refs) + 4  # the sweep gives many different dead sets
    dead, terr, score = gb.final_status()
    assert not dead.any()
    np.testing.assert_array_equal(score, gb.tt_score())
    for g, r in enumerate(refs):
        et, es = ref_tt_territory(r)
        np.testing.assert_array_equal(terr[g], et)
        assert es == score[g] == r.tt_score()
    e = gb.new_like(2)  # the empty board: score 0, every point dame
    d, t, s = e.final_status(np.zeros((2, 2, n * n), np.int32), 3, 0.5)
    assert (s == 0).all() and (t == 3).all() and not d.any()
    e.close()


# ---- the constructed 9x9 endgame ---------------------------------------------------------------------------
def endgame_9():
    """(black, white, dead) actions of a 9x9 endgame: black owns columns A-D with two eyes, white columns F-J with
    two eyes, column E is open, and one white stone sits at B5 inside black's area with its four liberties"""
    n = 9
    a = lambda x, y: x * n + y  # noqa: E731
    hole = {a(0, 1), a(0, 7), a(1, 4), a(1, 3), a(1, 5), a(0, 4), a(2, 4)}
    black = [a(x, y) for x in range(4) for y in range(n) if a(x, y) not in hole]
    white = [a(x, y) for x in range(5, 9) for y in range(n) if a(x, y) not in (a(8, 1), a(8, 7))] + [a(1, 4)]
    return black, white, [a(1, 4)]


def play_endgame(console):
    """enter the endgame with GTP play commands (a side with no stone left passes) and pass twice"""
    from elf_b200 import online

    black, white, _ = endgame_9()
    out = []
    for i in range(max(len(black), len(white))):
        for col, lst in (("B", black), ("W", white)):
            v = online.action2vertex(lst[i], 9) if i < len(lst) else "pass"
            out.append(console.execute(f"play {col} {v}"))
    out += [console.execute("play B pass"), console.execute("play W pass")]
    assert all(o == "=\n\n" for o in out), [o for o in out if o != "=\n\n"][:3]


def run_gtp_final_status(g, console):
    from elf_b200 import online

    black, white, dead = endgame_9()
    play_endgame(console)
    assert g.finished and g.finished[-1][2] == "two_pass"
    assert int(g.info()[0]) == 1 and not g.board.stones()[0].any()  # restarted: the kept position is used
    d = console.execute("final_status_list dead")
    al = console.execute("final_status_list alive")
    assert d == "= " + " ".join(online.action2vertex(a, 9) for a in dead) + "\n\n"
    alive_stones = sorted(v for line in al[2:].strip().split("\n") for v in line.split())
    assert alive_stones == sorted(online.action2vertex(a, 9) for a in black + white if a not in dead)
    assert console.execute("final_status_list seki") == "=\n\n"
    assert console.execute("final_status_list bogus").startswith("?")
    assert console.execute("final_status_list").startswith("?")
    assert "final_status_list" in console.commands
    return d, al


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


@pytest.mark.parametrize("n,K", [(9, 3), (19, 2)])
def test_ownership_and_final_status_equal_reference(emu, lane_order, n, K):
    need_ref(n)
    gb, refs, counts, K = run_ownership_equals_reference(emu.emu_batch, n, K, seed=11, order=lane_order)
    run_final_status_equals_reference(gb, refs, counts, K)


def test_ownership_arguments(emu):
    L = emu.emu_lib()
    gb = emu.emu_batch(3, 9)
    c = np.zeros((3, 2, 81), np.int32)
    for fn, extra in ((L.elfb200_ownership, (None, None)), (L.elfb200_ownership_dev, ())):
        assert fn(None, 1, 0, 10, c.ctypes.data, *extra) == ERR_ARG
        assert fn(gb._ctx, 1, 0, 10, None, *extra) == ERR_ARG
        assert fn(gb._ctx, 0, 0, 10, c.ctypes.data, *extra) == ERR_ARG
        assert fn(gb._ctx, -4, 0, 10, c.ctypes.data, *extra) == ERR_ARG
        assert fn(gb._ctx, 2 ** 30, 0, 10, c.ctypes.data, *extra) == ERR_ARG
        assert b"INT32_MAX" in L.elfb200_last_error()
        assert fn(gb._ctx, 1, 0, -1, c.ctypes.data, *extra) == ERR_ARG
    out = np.zeros((3, 81), np.uint8)
    assert L.elfb200_final_status(None, None, 1, 0.5, out.ctypes.data, None, None) == ERR_ARG
    assert L.elfb200_final_status(gb._ctx, c.ctypes.data, 0, 0.5, None, None, None) == ERR_ARG
    for bad in (float("nan"), float("inf"), float("-inf")):
        assert L.elfb200_final_status(gb._ctx, None, 1, bad, None, None, None) == ERR_ARG
    n0 = gb.launch_count()
    c[:] = 7
    assert L.elfb200_ownership_dev(gb._ctx, 2, 0, 0, c.ctypes.data) == 0  # zeroes the counts, counts the launch
    assert gb.launch_count() == n0 + 1
    assert (c[:, 1] == 0).all() and (c[:, 0] == 0).all()  # empty boards, no move: every point is dame
    assert L.elfb200_final_status(gb._ctx, None, 0, 0.5, None, None, None) == 0  # K is unused without counts
    assert gb.launch_count() == n0 + 2
    gb.close()


def test_online_final_status_uses_the_kept_position(emu):
    g, console = make_console(emu, 9)
    need_ref(9)
    black, white, dead = endgame_9()
    play_endgame(console)
    dead_groups, alive_groups = g.final_status(playouts=64, seed=1)
    assert dead_groups == [dead]
    assert sorted(a for grp in alive_groups for a in grp) == sorted(a for a in black + white if a not in dead)
    assert [grp[0] for grp in alive_groups] == sorted(grp[0] for grp in alive_groups)
    # the kept position is the reference's final position
    r = oracles.Ref(9)
    _replay_endgame(r)
    np.testing.assert_array_equal(g._final.stones()[0], r.stones())
    assert int(g._final.getHashCode()[0]) == r.hash()
    # once a move is played the current position is used
    console.execute("play B E5")
    dg, ag = g.final_status(playouts=16, seed=1)
    assert dg == [] and ag == [[4 * 9 + 4]]


def _replay_endgame(r):
    black, white, _ = endgame_9()
    for i in range(max(len(black), len(white))):
        r.forward(black[i] if i < len(black) else 81)
        r.forward(white[i] if i < len(white) else 81)
    r.forward(81)
    r.forward(81)


def test_gtp_final_status_list(emu):
    need_ref(9)
    g, console = make_console(emu, 9)
    console.final_status_playouts = 64
    run_gtp_final_status(g, console)
