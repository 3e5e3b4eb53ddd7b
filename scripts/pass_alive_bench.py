#!/usr/bin/env python
"""Pass-alive chains and areas (elfb200_pass_alive_dev, k_pass_alive) on the H100.  Prints one JSON line per
workload with the card's name and power limit, read in the same run.

Workloads:
  end19   4096 19x19 terminal positions of the eye-avoiding random policy (tests/test_pass_alive.py's games)
  mid19   4096 19x19 positions 150 plies into games of the same policy
  end9    16,384 9x9 terminal positions of that policy
  gtp     one 19x19 terminal position through final_status(pass_alive=True), the GTP final_status_list case

  call_us        device events around back-to-back elfb200_pass_alive_dev calls (after warm-up), per call; for
                 gtp, a host clock around whole synchronous final_status(pass_alive=True) calls without counts
  alive_stones   stones of pass-alive chains, both colours, over the batch
  area_points    points of either colour's pass-alive area over the batch"""
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import test_pass_alive as TP  # noqa: E402


def gpu_name_and_power():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return name, power


def positions(n, G, max_plies, seed):
    """move lists of G games of the eye-avoiding random policy, played in worker processes"""
    chunk = 128
    jobs = [(n, seed * 100003 + i, min(chunk, G - i), max_plies) for i in range(0, G, chunk)]
    with mp.get_context("fork").Pool(min(len(jobs), os.cpu_count() or 1)) as pool:
        parts = pool.map(_lists, jobs)
    return [m for p in parts for m in p]


def _lists(args):
    n, seed, count, max_plies = args
    rng = np.random.default_rng(seed)
    return [TP.eye_avoiding_game(n, rng, max_plies=max_plies)[0] for _ in range(count)]


def bench(label, n, lists, iters, name, power):
    import torch

    from elf_b200.board import GoBatch

    gb = GoBatch(len(lists), board_size=n)
    gb.replay(lists)
    alive, area = gb.pass_alive()
    at = torch.empty(alive.shape, dtype=torch.uint8, device="cuda")
    rt = torch.empty_like(at)
    for _ in range(3):
        gb.pass_alive(out=(at, rt))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        gb.pass_alive(out=(at, rt))
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000.0 / iters
    assert (at.cpu().numpy() == alive).all() and (rt.cpu().numpy() == area).all(), "device and host forms differ"
    print(json.dumps({"workload": label, "games": len(lists), "call_us": round(us, 1),
                      "alive_stones": int(alive.sum()), "area_points": int((area > 0).sum()),
                      "gpu": name, "power_limit": power}), flush=True)
    gb.close()


def bench_gtp(lists, iters, name, power):
    import torch

    from elf_b200.board import GoBatch

    gb = GoBatch(1, board_size=19)
    gb.replay(lists[:1])
    alive, area = gb.pass_alive()
    for _ in range(5):
        gb.final_status(pass_alive=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        gb.final_status(pass_alive=True)  # synchronous: ends in a stream synchronise
    us = (time.perf_counter() - t0) * 1e6 / iters
    print(json.dumps({"workload": "gtp", "games": 1, "call_us": round(us, 1), "alive_stones": int(alive.sum()),
                      "area_points": int((area > 0).sum()), "gpu": name, "power_limit": power}), flush=True)
    gb.close()


def main():
    end19 = positions(19, 4096, None, seed=1)
    mid19 = positions(19, 4096, 150, seed=2)
    end9 = positions(9, 16384, None, seed=3)
    name, power = gpu_name_and_power()
    bench("end19", 19, end19, 50, name, power)
    bench("mid19", 19, mid19, 50, name, power)
    bench("end9", 9, end9, 50, name, power)
    bench_gtp(end19, 200, name, power)


if __name__ == "__main__":
    main()
