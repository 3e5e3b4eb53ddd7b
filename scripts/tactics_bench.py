#!/usr/bin/env python
"""Ladders and self-ataris (elfb200_tactics_dev, k_tactics) on the H100.  Prints one JSON line per workload with
the card's name and power limit, read in the same run.

Workloads:
  random19     4096 19x19 positions about 150 plies into random games (GoEnv + random_legal_actions)
  ladder_suite the 12,522 positions of tests/golden/ladder_suite.json.gz (the reference's ladder_suite/ games)
               in one batch

  ladder_us     device events around back-to-back elfb200_tactics_dev calls (after warm-up) with only the
                ladder output, per call
  both_us       the same with ladder and self_atari
  searched      (position, point, colour) triples whose ladder search ran (calls > 0, from the host form)
  ladders       triples with a ladder (depth > 0)
  search_calls  checkLadderUseSearch calls of all searches together; max_calls the largest for one triple"""
import gzip
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elf_b200.board import GoBatch  # noqa: E402
from elf_b200.env import GoEnv, random_legal_actions  # noqa: E402
from elf_b200 import sgf  # noqa: E402

DEV = torch.device("cuda", 0)


def gpu_name_and_power():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return name, power


def ladder_suite_lists():
    """the move list of every prefix of every record of the ladder suite"""
    lists = []
    path = os.path.join(ROOT, "tests", "golden", "ladder_suite.json.gz")
    for rec in json.load(gzip.open(path, "rt"))["records"]:
        moves = []
        for m in sgf.Sgf.loads(rec["sgf"]):
            if m.action < 0:
                break
            moves.append(int(m.action))
            lists.append(list(moves))
    return lists


def random_positions(G, n, plies, seed):
    env = GoEnv.create(G, board_size=n)
    obs = env.reset()
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    for _ in range(plies):
        obs = env.step(random_legal_actions(obs["legal"], counter, seed=seed))
    torch.cuda.synchronize()
    return env, env.board


def time_dev(gb, out, iters):
    for _ in range(3):
        gb.tactics(out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        gb.tactics(out=out)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / iters


def bench(label, gb, iters, name, power):
    n, G = gb.board_size, gb.num_games
    lad, sa, calls = gb.tactics(trace=True)
    lt = torch.empty((G, 2, n * n), dtype=torch.int16, device=DEV)
    st = torch.empty_like(lt)
    ladder_us = time_dev(gb, (lt, None), iters)
    both_us = time_dev(gb, (lt, st), iters)
    assert (lt.cpu().numpy() == lad).all() and (st.cpu().numpy() == sa).all(), "device and host forms differ"
    print(json.dumps({"workload": label, "games": G, "ladder_us": round(ladder_us, 1), "both_us": round(both_us, 1),
                      "searched": int((calls > 0).sum()), "ladders": int((lad > 0).sum()),
                      "search_calls": int(calls.astype(np.int64).sum()), "max_calls": int(calls.max()),
                      "max_depth": int(lad.max()), "self_ataris": int((sa > 0).sum()),
                      "gpu": name, "power_limit": power}), flush=True)


def main():
    name, power = gpu_name_and_power()
    env, gb = random_positions(4096, 19, 150, seed=3)
    bench("random19", gb, 20, name, power)
    env.close()
    lists = ladder_suite_lists()
    gb = GoBatch(len(lists), board_size=19)
    gb.replay(lists)
    bench("ladder_suite", gb, 20, name, power)
    gb.close()


if __name__ == "__main__":
    main()
