#!/usr/bin/env python
"""Monte-Carlo ownership (elfb200_ownership_dev, k_ownership) and dead stones (elfb200_final_status) on the H100.
Prints one JSON line per workload with the card's name and power limit, read in the same run.

Workloads:
  19x19   4096 positions about 150 plies in (GoEnv + random_legal_actions), K = 16 playouts each
  9x9     12,288 positions at ply 40, K = 8
  gtp     one 19x19 position, K = 1024, then final_status: what a GTP controller's final_status_list costs

  own_us        device events around back-to-back elfb200_ownership_dev calls (after warm-up), per call
  moves_per_s   playout moves of one traced call (sum of plies) over own_us
  status_us     (gtp) host clock around GoBatch.final_status with the counts, per call
  checksum      sum of counts * (index + 1) mod 2^61 - 1, equal between two runs in this call"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elf_b200.board import GoBatch  # noqa: E402
from elf_b200.env import GoEnv, random_legal_actions  # noqa: E402

DEV = torch.device("cuda", 0)


def gpu_name_and_power():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return name, power


def positions(G, n, plies, seed):
    """G positions `plies` steps of the seeded uniform policy into GoEnv (a game that ends restarts)"""
    env = GoEnv.create(G, board_size=n)
    obs = env.reset()
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    for _ in range(plies):
        obs = env.step(random_legal_actions(obs["legal"], counter, seed=seed))
    torch.cuda.synchronize()
    return env


def checksum(counts):
    c = counts.astype(np.int64).ravel()
    return int((c * (np.arange(c.size, dtype=np.int64) % 1000003 + 1)).sum() % ((1 << 61) - 1))


def bench(gb, K, iters):
    n = gb.board_size
    out = torch.empty((gb.num_games, 2, n * n), dtype=torch.int32, device=DEV)
    counts, _, plies = gb.ownership(K, seed=1, trace=True)  # also allocates the scratch
    for _ in range(3):
        gb.ownership(K, seed=1, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        gb.ownership(K, seed=1, out=out)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000.0 / iters
    again = out.cpu().numpy()
    assert (again == counts).all(), "counts differ between two runs"
    return us, int(plies.astype(np.int64).sum()), counts


def main():
    name, power = gpu_name_and_power()
    for label, n, G, plies, K, iters in (("19x19", 19, 4096, 150, 16, 5), ("9x9", 9, 12288, 40, 8, 10)):
        env = positions(G, n, plies, seed=3)
        us, moves, counts = bench(env.board, K, iters)
        print(json.dumps({"workload": label, "games": G, "playouts": K, "own_us": round(us, 1),
                          "moves": moves, "moves_per_s": round(moves / (us * 1e-6)),
                          "checksum": checksum(counts), "gpu": name, "power_limit": power}), flush=True)
        env.close()
    env = positions(1, 19, 200, seed=5)
    src = env.board
    gb = GoBatch(1, board_size=19)
    gb.gather(src, [0])
    us, moves, counts = bench(gb, 1024, 20)
    gb.final_status(counts, 1024, 0.5)
    t0 = time.perf_counter()
    for _ in range(20):
        dead, _, score = gb.final_status(counts, 1024, 0.5)
    st_us = (time.perf_counter() - t0) * 1e6 / 20
    print(json.dumps({"workload": "gtp", "games": 1, "playouts": 1024, "own_us": round(us, 1), "moves": moves,
                      "moves_per_s": round(moves / (us * 1e-6)), "status_us": round(st_us, 1),
                      "dead_stones": int(dead.sum()), "score": int(score[0]), "checksum": checksum(counts),
                      "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
