#!/usr/bin/env python
"""Copying games between batches (elfb200_gather_games_dev, k_gather) and a one-ply lookahead round built on
it, on the H100.  Prints one JSON line with the card's name and power limit, read in the same run.

Configurations: 4096 19x19 source games at ply ~150 copied into 32,768 branch slots (K = 8), and 12,288 9x9
source games at ply ~60 into 49,152 slots (K = 4); index = arange(G).repeat_interleave(K).

  gather_us      device events around 200 back-to-back elfb200_gather_games_dev calls on the destination
                 stream (after 20 warm-up calls), per call
  moved_MB       bytes the copy must move: every destination game written once (2.35 KB on 19x19 plus 8 B
                 per recorded move), every source game read once (its K copies read it again from L2)
  hbm_frac       moved bytes / gather time over the HBM peak (MEASURED_PEAKS.json's hbm_gbs if present, else
                 the H100 SXM data sheet's 3.35 TB/s)
  round_*_us     one lookahead round: GoEnv.load of the K branches, a random legal action per branch,
                 GoEnv.step with fp16 planes, the best branch per game by value (captures break ties), and
                 GoEnv.load of the chosen branch back into the root env; eager, and as a CUDA graph of
                 16 rounds replayed (device events, warmed up)"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elf_b200 import lib as _l  # noqa: E402
from elf_b200.env import GoEnv, random_legal_actions  # noqa: E402

_PEAKS = os.path.join(ROOT, "MEASURED_PEAKS.json")
PEAK_GBS = json.load(open(_PEAKS))["hbm_gbs"] if os.path.exists(_PEAKS) else 3350.0  # H100 SXM data sheet (HBM3)
DEV = torch.device("cuda", 0)


def gpu_name_and_power():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return name, power


def play(env, plies, seed):
    """plies of the seeded uniform policy; returns the number of recorded (non-pass) moves of every game"""
    P = env.board_size ** 2
    obs = env.reset()
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    nsk = torch.zeros(env.num_games, dtype=torch.int64, device=DEV)
    for _ in range(plies):
        a = random_legal_actions(obs["legal"], counter, seed=seed)
        obs = env.step(a)
        nsk = torch.where(obs["done"].bool(), 0, nsk + ((obs["ok"] == 1) & (a != P)).long())
    return nsk


def game_bytes(n):
    """bytes of one stored game besides its superko record (k_gather: cur, sa, ring, legal, placed, hash,
    meta, sk_n)"""
    return 8 * n + 8 * n + 64 * n + 4 * n + 2 * n * n + 8 + 16 + 4


def time_gather(dst, src, idx, reps=200):
    L = dst._lib
    st = torch.cuda.ExternalStream(dst.stream, device=DEV)
    for _ in range(20):
        _l.check(L, L.elfb200_gather_games_dev(dst._ctx, src._ctx, idx.data_ptr()))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(reps):
        _l.check(L, L.elfb200_gather_games_dev(dst._ctx, src._ctx, idx.data_ptr()))
    e1.record(st)
    e1.synchronize()
    return 1e3 * e0.elapsed_time(e1) / reps


def lookahead_round(root, branch, idx, K, counter):
    G = root.num_games
    bobs = branch.load(root, idx)
    bobs = branch.step(random_legal_actions(bobs["legal"], counter, seed=7))
    info = bobs["info"]
    score = bobs["value"] + 1e-3 * (info[:, 2] - info[:, 3]).float()  # black's view
    score = torch.where(root.info[:, 1].repeat_interleave(K) == 1, score, -score)  # the root's side to move
    best = score.view(G, K).argmax(1)
    chosen = (torch.arange(G, device=DEV) * K + best).to(torch.int32)
    return root.load(branch, chosen)


def time_rounds(root, branch, idx, K, graph, rounds=16, reps=5):
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    for _ in range(3):
        lookahead_round(root, branch, idx, K, counter)
    torch.cuda.synchronize()
    cur = torch.cuda.current_stream(DEV)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(rounds):
                lookahead_round(root, branch, idx, K, counter)
        g.replay()
        torch.cuda.synchronize()
        e0.record(cur)
        for _ in range(reps):
            g.replay()
        e1.record(cur)
    else:
        e0.record(cur)
        for _ in range(reps * rounds):
            lookahead_round(root, branch, idx, K, counter)
        e1.record(cur)
    e1.synchronize()
    return 1e3 * e0.elapsed_time(e1) / (reps * rounds)


def run(n, G, K, plies):
    root = GoEnv.create(G, board_size=n, features="f16")
    nsk = play(root, plies, seed=3)
    branch = GoEnv.create(K * G, board_size=n, features="f16")
    idx = torch.arange(G, device=DEV, dtype=torch.int32).repeat_interleave(K)
    gb, sb = game_bytes(n), 8 * nsk
    moved = K * (G * gb + int(sb.sum())) + (G * gb + int(sb.sum()))
    us = time_gather(branch.board, root.board, idx)
    torch.cuda.synchronize()
    assert (branch.board.getHashCode() == root.board.getHashCode()[idx.cpu().numpy()]).all()
    plies_now = root.board.getPly()
    res = {"board": n, "src_games": G, "K": K, "dst_games": K * G, "mean_ply": round(float(plies_now.mean()), 1),
           "mean_recorded_moves": round(float(nsk.float().mean()), 1), "gather_us": round(us, 2),
           "moved_MB": round(moved / 1e6, 1), "moved_GBs": round(moved / us / 1e3, 1),
           "hbm_frac": round(moved / us / 1e3 / PEAK_GBS, 3)}
    # the lookahead rounds change the root positions: time them after the copy measurement
    res["round_eager_us"] = round(time_rounds(root, branch, idx, K, graph=False), 1)
    res["round_graph_us"] = round(time_rounds(root, branch, idx, K, graph=True), 1)
    root.close()
    branch.close()
    return res


def main():
    name, power = gpu_name_and_power()
    out = {"gpu": name, "power_limit": power, "hbm_peak_gbs": PEAK_GBS,
           "runs": [run(19, 4096, 8, 150), run(9, 12288, 4, 60)]}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
