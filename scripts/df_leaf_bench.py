#!/usr/bin/env python
"""Times the search's leaf-plane writers on one wave of pending leaves: the DarkForest writer
(k_leaf_features_df, ELFB200_FEAT_DF_F32_NCHW) and the AGZ float32 writer (k_leaf_features,
ELFB200_FEAT_F32_NCHW), alternated in the same run.

4096 games of 19x19 at 800 rollouts (the benchmark's search), 16 random opening plies, a few waves of
search with a hash-keyed fake network so the trees have depth, then device events around 10 back-to-back
elfb200_mcts_leaf_features calls per writer on the last wave's pending leaves.  Prints the card name and
power limit, ms per wave and the bytes written (DF: 25 planes * 361 * 4 B = 36,100 B per position, plus the
parent-chain reads; AGZ: 25,992 B).  Needs a CUDA device; writes nothing.

    python scripts/df_leaf_bench.py [--games 4096] [--waves 40] [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=4096)
    ap.add_argument("--board", type=int, default=19, choices=[9, 19])
    ap.add_argument("--rollouts", type=int, default=800)
    ap.add_argument("--waves", type=int, default=40, help="waves searched before the timed one")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the two writers")
    args = ap.parse_args()

    import numpy as np
    import torch

    import elf_b200
    from elf_b200 import lib as _l
    from tests.planenet import fakenet_torch
    from tests.search_scale import random_opening

    if not torch.cuda.is_available():
        raise SystemExit("df_leaf_bench needs a CUDA device")
    n, G = args.board, args.games
    gb = elf_b200.GoBatch(G, board_size=n)
    random_opening([gb], 16, np.random.default_rng(1))
    mc = elf_b200.MctsBatch(gb, feature_format="df", rotation_flip=1, num_rollouts=args.rollouts,
                            num_rollouts_per_batch=8, virtual_loss=1, persistent_tree=1, c_puct=1.5)

    def net(batch):  # priors and values from the leaves' planes (no host round trip)
        x = batch["s"]
        key = x.flatten(1).view(torch.int32).to(torch.int64).sum(1)
        pi, v = fakenet_torch(key, n * n + 1)
        return {"pi": pi, "V": v}

    mc.begin_move()
    for _ in range(args.waves):
        mc.wave(net)
    s = mc.select()  # the timed wave: its leaves stay pending
    k = s.shape[0]
    df = mc.feat
    agz = torch.empty((mc.max_leaves, 18, n, n), dtype=torch.float32, device=mc.device)
    L, m = mc._lib, mc._m
    stream = torch.cuda.ExternalStream(gb.stream, device=mc.device)

    def timed(buf, fmt):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        with torch.cuda.stream(stream):
            ev[0].record(stream)
            for _ in range(args.reps):
                _l.check(L, L.elfb200_mcts_leaf_features(m, buf.data_ptr(), fmt, 0))
            ev[1].record(stream)
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1]) / args.reps

    timed(df, _l.FEAT_DF_F32_NCHW)
    timed(agz, _l.FEAT_F32_NCHW)
    t_df, t_agz = [], []
    for _ in range(args.rounds):
        t_df.append(timed(df, _l.FEAT_DF_F32_NCHW))
        t_agz.append(timed(agz, _l.FEAT_F32_NCHW))
    ok = torch.equal(df[:k], s)  # the repeated writes are the select's planes
    P = n * n
    out = {"card": card(), "games": G, "board": n, "rollouts": args.rollouts, "leaves": k,
           "df_ms_per_wave": float(np.median(t_df)), "agz_f32_ms_per_wave": float(np.median(t_agz)),
           "df_bytes_written": k * 25 * P * 4, "agz_bytes_written": k * 18 * P * 4,
           "df_GBps": k * 25 * P * 4 / (np.median(t_df) * 1e6), "agz_GBps": k * 18 * P * 4 / (np.median(t_agz) * 1e6),
           "df_spread_ms": [float(min(t_df)), float(max(t_df))], "agz_spread_ms": [float(min(t_agz)), float(max(t_agz))],
           "idempotent": bool(ok)}
    print(json.dumps(out), flush=True)
    mc.close()
    gb.close()


if __name__ == "__main__":
    main()
