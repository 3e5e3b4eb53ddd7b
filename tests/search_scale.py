"""The self-play search at the benchmark's own size, as one scenario with pluggable back ends (test
infrastructure only).

``run_scale`` plays the bench's workload on G games split into parts: 16 seeded random opening plies
(``bench.random_opening``'s rule), then K searched moves.  Each move is searched by ``drive`` (the caller
picks ``WavePipeline``, the product's ``MctsBatch.search`` or ``padded_search``), chosen on the device by
``choose(policy_distri_cutoff=0, resign_thres=0)``, played with ``GoBatch.forward`` and followed by
``advance``.  The searches' network is a ``tests.planenet.PlaneNet``, a pure function of the leaf planes.

A sample of the games is mirrored on host states (``oracles.Oracle`` / ``oracles.Ref``) and searched by
a CPU search (``oracles.OracleMcts`` / ``oracles.RefMcts``) on the numpy twin of the same net; every
move of those games is compared with the device's.  The root tables of all games are returned, so two
layouts of the same games can be compared bitwise.

The GPU tests (``tests/test_zz_gpu_search_at_scale.py``) run it on an H100; ``tests/test_search_scale.py``
runs the same function on the SIMT emulator build at a small size."""
import numpy as np

OPENING_PLIES = 16


def part_sizes(G, parts):
    """bench.SelfPlayEngine's split of G games into parts"""
    return [G // parts + (1 if i < G % parts else 0) for i in range(parts)]


def sample_games(G, parts, count=32, seed=0):
    """the first, second, 32nd and 33rd games, both sides of every part boundary, the last game, and
    seeded random games up to ``count``"""
    bounds = np.cumsum(part_sizes(G, parts))[:-1]
    fixed = {0, 1, 31, 32, G // 2 - 1, G // 2, G - 1} | {int(b) - 1 for b in bounds} | {int(b) for b in bounds}
    fixed = {g for g in fixed if 0 <= g < G}
    rng = np.random.default_rng(seed)
    rest = [g for g in rng.permutation(G) if g not in fixed]
    return sorted(fixed | set(int(g) for g in rest[: max(0, count - len(fixed))]))


def random_opening(boards, plies, rng):
    """``plies`` uniformly random legal non-pass moves in every game, drawn over the concatenation of
    the parts (so the games do not depend on the split); a game without a legal point passes.
    Returns int32 [plies, G], the moves played."""
    n = boards[0].board_size
    played = []
    for _ in range(plies):
        lg = np.concatenate([gb.legal_mask()[:, :-1] for gb in boards]).astype(np.float64)
        tot = lg.sum(1, keepdims=True)
        c = (lg / np.maximum(tot, 1)).cumsum(1)
        a = np.minimum((c < rng.random((lg.shape[0], 1))).sum(1), n * n - 1).astype(np.int32)
        a[tot[:, 0] == 0] = n * n
        lo = 0
        for gb in boards:
            assert gb.forward(a[lo: lo + gb.num_games]).all()
            lo += gb.num_games
        played.append(a)
    return np.stack(played)


def padded_search(searches, net):
    """``MctsBatch.search`` for each part in turn, with ``wave_select``'s padding of the leaf batch to a
    multiple of ``net.batchsize`` (rows past the leaf count are stale; their replies must be ignored).
    For the emulator build, whose search class has no padding of its own."""
    pad = int(getattr(net, "batchsize", 0) or 0)
    for s in searches:
        s.begin_move()
        for _ in range(s.waves_per_move):
            x = s.select()
            k = x.shape[0]
            if k == 0:
                s.expand_backup(None, None)
                continue
            if pad > 1:
                x = s.feat[: min(-(-k // pad) * pad, s.max_leaves)]
            r = net({s.feat_key: x})
            s.expand_backup(r["pi"], r["V"])


def run_scale(make_board, make_search, drive, net, n, G, parts, moves, sample=(), make_state=None,
              make_cpu=None, tol=0, seed=20260922, close=True):
    """The scenario described in the module docstring.

    make_board(G_part) -> GoBatch; make_search(gb, first_game) -> search; drive(searches, net): one move's
    search of every part; make_state() -> host state; make_cpu(g) -> CPU search of game g (its ``act``
    runs on ``planenet.callback``).  ``tol``: allowed |visit difference| per edge against the CPU search
    (0 = equal tables, equal moves, equal root values bit for bit).  Where a table is not exact and the
    moves differ, both sides play the CPU's move.

    Returns a dict: per-move tables of all games ("visits" [K,G,A] int32, "root_value", "best_q",
    "total_visits", "action" (the device's choice), "best_action"), "evals", "errors", "stats", and for
    the sample "compared", "exact", "worst", "ended" (games that reached a terminal root, not compared)."""
    sizes = part_sizes(G, parts)
    boards, searches = [], []
    try:
        boards += [make_board(g) for g in sizes]
        return _run(boards, searches, make_search, drive, net, G, moves, sample, make_state, make_cpu, tol, seed)
    finally:
        if close:  # also when an assertion fails: a full-size node pool must not outlive its test
            for s in searches:
                s.close()
            for gb in boards:
                gb.close()


def _run(boards, searches, make_search, drive, net, G, moves, sample, make_state, make_cpu, tol, seed):
    sizes = [gb.num_games for gb in boards]
    firsts = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(int)
    rng = np.random.default_rng(seed)
    opening = random_opening(boards, OPENING_PLIES, rng)
    searches += [make_search(gb, int(lo)) for gb, lo in zip(boards, firsts)]
    sample = list(sample)
    states = {g: make_state() for g in sample}
    cpu = {g: make_cpu(g) for g in sample}
    for g in sample:
        for a in opening[:, g]:
            assert states[g].forward(int(a))
    out = {k: [] for k in ("visits", "root_value", "best_q", "total_visits", "action", "best_action")}
    compared = exact = worst = 0
    ended = set()
    for mv in range(moves):
        drive(searches, net)
        res = [s.results() for s in searches]
        acts = np.concatenate([s.choose(0, 0.0)[0] for s in searches])
        for k in ("visits", "root_value", "best_q", "total_visits", "best_action"):
            out[k].append(np.concatenate([r[k] for r in res]))
        out["action"].append(acts.copy())
        vis = out["visits"][-1]
        searched = acts >= 0
        np.testing.assert_array_equal(acts[searched], out["best_action"][-1][searched], err_msg=f"move {mv}")
        for g in sample:
            st = states[g]
            if st.terminated():
                ended.add(g)
                assert acts[g] < 0, f"move {mv} game {g}: a finished game was searched"
                continue
            rr = cpu[g].act(st)
            tag = f"move {mv} game {g}"
            gv, rv = vis[g], rr["visits"]
            assert ((gv >= 0) == (rv >= 0)).all(), f"edge sets differ: {tag}"
            d = int(np.abs(gv - rv)[rv >= 0].max())
            worst, compared, exact = max(worst, d), compared + 1, exact + (d == 0)
            assert d <= tol, f"visits differ by {d} at {tag}"
            assert out["total_visits"][-1][g] == rr["total_visits"], tag
            if tol == 0:
                assert out["root_value"][-1][g].tobytes() == np.float32(rr["root_value"]).tobytes(), \
                    f"root_value {out['root_value'][-1][g]!r} != {rr['root_value']!r}: {tag}"
            if d == 0:
                assert acts[g] == rr["best_action"], f"move {acts[g]} != {rr['best_action']}: {tag}"
                assert abs(out["best_q"][-1][g] - rr["best_q"]) < 1e-5, tag
            else:
                acts[g] = rr["best_action"]
            assert st.forward(int(acts[g])), tag
        for gb, s, lo in zip(boards, searches, firsts):
            a = acts[lo: lo + gb.num_games]
            assert gb.forward(a)[a >= 0].all(), f"move {mv}"
            s.advance(a)
    out = {k: np.stack(v) for k, v in out.items()}
    out["evals"] = sum(int(s.eval_count()) for s in searches)
    out["errors"] = np.sum([s.errors() for s in searches], axis=0)
    out["stats"] = np.sum([s.stats() for s in searches], axis=0)
    out.update(compared=compared, exact=exact, worst=worst, ended=sorted(ended))
    return out


def assert_same_tables(a, b, label):
    """two runs of the same games: every table of every game at every move bitwise equal"""
    for k in ("visits", "total_visits", "action", "best_action"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=f"{label}: {k}")
    for k in ("root_value", "best_q"):
        bad = np.argwhere(a[k].view(np.uint32) != b[k].view(np.uint32))
        assert len(bad) == 0, f"{label}: {k} differs at (move, game) {bad[:8].tolist()}"
    assert a["evals"] == b["evals"], (label, a["evals"], b["evals"])


def summary(name, r, extra=""):
    e, s = r["errors"], r["stats"]
    return (f"[{name}] compared {r['compared']} game-moves, exact tables {r['exact']}, worst deviation {r['worst']}, "
            f"ended {len(r['ended'])}; evals {r['evals']}; errors {e.tolist()}; stats (descent steps, edge records "
            f"read, nodes created, stored edges of visited nodes) {s.tolist()}{extra}")


def check_net(net):
    """the digest net saw only values in {0, 1} over the whole run (one read of the device counter)"""
    bad = int(net.bad.item())
    assert bad == 0, f"{bad} plane values outside {{0, 1}} reached the network"
    assert net.calls > 0
