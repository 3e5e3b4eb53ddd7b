#!/usr/bin/env python
"""Microseconds per ply of a batch of games driven from the device (elf_b200.env.GoEnv) against the
host-driven step API, on 4096 19x19 and 12,288 9x9 games.  Prints one JSON line with the card's name and
power limit, read in the same run.

Modes per size (device events, every mode warmed up first):
  host_step_us   (a) GoBatch.forward (elfb200_step: host actions in, accept flags out, one wait per ply),
                     the golden playout's move sequence played by every game, as scripts/step_probe.py does
  env_eager_us   (b) random_legal_actions -> GoEnv.step, no planes, launched eagerly
  env_f16_us     (c) (b) with fp16 NHWC planes written after every step
  env_graph_us   (d) (c) captured once as a CUDA graph of 64 plies and replayed
  *_no_policy_us     the same mode playing the actions logged in its first run again, without the policy
                     (graph: one graph over all timed plies): what the env itself costs per ply
Each of (b)-(d) also adds the step's values into a float64 accumulator per ply (one small kernel), and
plays the same plies from the same seed: the run checks that their final hashes and value sums agree.
The policy draws uniformly among all legal moves (the env has no eye mask), so games fill their eyes
and often run to the 2N^2 ply cap; every way a game can end occurs."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import elf_b200  # noqa: E402
from elf_b200.env import GoEnv, random_legal_actions  # noqa: E402

GRAPH_PLIES = 64


def gpu_name_and_power():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return name, power


def host_step(G, n):
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", f"playouts_{n}.json")))
    mv = next(e["moves"] for e in gold["games"] if "moves" in e)
    gb = elf_b200.GoBatch(G, board_size=n)
    acts = np.empty(G, np.int32)
    for rep in range(2):  # the first pass warms up
        gb.reset()
        t0 = time.perf_counter()
        for a in mv:
            acts.fill(a)
            ok = gb.forward(acts)
        dt = time.perf_counter() - t0
    assert ok.all()
    gb.close()
    return 1e6 * dt / len(mv)


def env_run(G, n, plies, mode, seed, log=None):
    """GRAPH_PLIES warm-up plies, then `plies` timed plies.  Without `log` the actions come from the seeded
    policy and are logged; with it, the logged actions are played again, which times the env alone.
    Returns (us per ply, final hashes, value sum, action log)."""
    env = GoEnv.create(G, board_size=n, features=None if mode == "eager" else "f16")
    counter = torch.zeros(1, dtype=torch.int64, device=env.device)
    vacc = torch.zeros(G, dtype=torch.float64, device=env.device)
    replay = log is not None
    if not replay:
        log = torch.empty((GRAPH_PLIES + plies, G), dtype=torch.int32, device=env.device)
    obs = env.reset()

    def ply(obs, t):
        if replay:
            a = log[t]
        else:
            a = random_legal_actions(obs["legal"], counter, seed)
            log[t].copy_(a)
        obs = env.step(a)
        vacc.add_(obs["value"])
        return obs

    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if mode == "graph":
        # the policy's first kernels run outside the capture, on a scratch state
        random_legal_actions(torch.ones_like(obs["legal"]), torch.zeros_like(counter))
        torch.cuda.synchronize()
        # with the policy: one graph of 64 plies, replayed (the log rows are a graph input, written in place);
        # replaying logged actions: the warm-up graph, then one graph over all timed plies
        warm, timed = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(warm):
            for t in range(GRAPH_PLIES):
                obs = ply(obs, t)
        if replay:
            with torch.cuda.graph(timed):
                for t in range(plies):
                    obs = ply(obs, GRAPH_PLIES + t)
        warm.replay()
        ev0.record()
        if replay:
            timed.replay()
        else:
            for _ in range(plies // GRAPH_PLIES):
                warm.replay()
        ev1.record()
    else:
        for t in range(GRAPH_PLIES):
            obs = ply(obs, t)
        ev0.record()
        for t in range(plies):
            obs = ply(obs, GRAPH_PLIES + t)
        ev1.record()
    torch.cuda.synchronize()
    us = 1e3 * ev0.elapsed_time(ev1) / plies
    h = env.board.getHashCode()
    vs = float(vacc.sum())
    env.close()
    return us, h, vs, log


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--plies", type=int, default=10 * GRAPH_PLIES, help="timed plies per mode (a multiple of 64)")
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    assert args.plies % GRAPH_PLIES == 0
    if not torch.cuda.is_available():
        sys.exit("env_bench needs a CUDA device")
    name, power = gpu_name_and_power()
    out = {"gpu": name, "power_limit": power, "timed_plies": args.plies, "warmup_plies": GRAPH_PLIES}
    for n, G in ((19, 4096), (9, 12288)):
        r = {"games": G, "host_step_us": round(host_step(G, n), 2)}
        ref = None
        for mode in ("eager", "f16", "graph"):
            us, h, vs, log = env_run(G, n, args.plies, mode, args.seed)
            r[f"env_{mode}_us"] = round(us, 2)
            if ref is None:
                ref = (h, vs, log)
                r["value_sum"] = vs
            assert (h == ref[0]).all() and vs == ref[1], f"{n}x{n} {mode}: final state differs from the eager run"
            # the same plies again from the logged actions: the env without the policy
            us, h, vs, _ = env_run(G, n, args.plies, mode, args.seed, log=ref[2])
            r[f"env_{mode}_no_policy_us"] = round(us, 2)
            assert (h == ref[0]).all() and vs == ref[1], f"{n}x{n} {mode}: replayed actions give another state"
        r["modes_agree"] = True
        out[f"{n}x{n}"] = r
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
