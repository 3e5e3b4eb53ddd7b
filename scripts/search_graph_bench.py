#!/usr/bin/env python
"""Moves per second of one AlphaZero-style self-play loop over GoEnv, driven three ways:
  (a) host:  MctsBatch.search / choose, GoBatch.forward, advance, reset -- the host waits for every wave's leaf
             count and reads every move's actions back;
  (b) dev:   the device forms (search_dev / choose_dev / advance_dev / reset_dev with GoEnv.step), eagerly;
  (c) graph: one such move captured in a torch.cuda.CUDAGraph and replayed.
The same network serves all three: FusedActor(cuda_graph=False) (a captured actor may not replay a graph of its own)
on the 16-bit channels-last leaf batch.  Configurations: 9x9 at G = 1024 and 19x19 at G = 512 with a 6x64 tower and
64 rollouts per move (8 per wave), and the benchmark's own (4096 x 19x19 x 800 rollouts, 20x256) for (a) and (b)
only, with a pool of 900 nodes per game (the default 1856 would take 56 GB per handle, and the two handles must
both fit the card).  Every form is warmed up on every shape first; the forms then alternate, timed with device
events.  Prints the card name and power limit, then one JSON line per configuration."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from elf_b200 import GoBatch  # noqa: E402
from elf_b200.env import GoEnv  # noqa: E402
from elf_b200.mcts import MctsBatch  # noqa: E402
from elf_b200.model import FusedActor, PolicyValueNet  # noqa: E402

CUTOFF, THRES, SEED = 30, 0.05, 1234 << 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


class HostLoop:
    def __init__(self, G, n, net, opts):
        self.gb = GoBatch(G, board_size=n, device=0)
        self.mc = MctsBatch(self.gb, feature_format="f16", **opts)
        self.net, self.k = net, 0

    def move(self):
        self.mc.search(self.net)
        a, _ = self.mc.choose(CUTOFF, THRES, seed=SEED ^ self.k)
        self.gb.forward(a)
        ended = (self.gb.terminated() | (a == -1)).astype("uint8")
        self.gb.reset(ended)
        self.mc.advance(a)
        self.mc.reset(ended)
        self.k += 1


class DevLoop:
    def __init__(self, G, n, net, opts):
        self.env = GoEnv.create(G, board_size=n, device=0, features=None)
        self.mc = MctsBatch(self.env.board, feature_format="f16", **opts)
        self.net = net
        self.move_t = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.graph = None

    def move(self):
        mc, env = self.mc, self.env
        mc.search_dev(self.net, self.move_t)
        a, _ = mc.choose_dev(CUTOFF, THRES, seed=self.move_t ^ SEED)
        obs = env.step(a)
        resigned = a == -1
        ended = obs["done"].bool() | resigned
        env.reset(resigned)
        mc.advance_dev(a)
        mc.reset_dev(ended)
        self.move_t.add_(1)

    def capture(self):
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.move()

    def replay(self):
        self.graph.replay()


def timed(fn, moves):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(moves):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3


def run(name, G, n, blocks, dim, rollouts, nn_batch, moves, rounds, graph, nodes_per_game=0):
    model = PolicyValueNet(n, num_block=blocks, dim=dim).cuda().eval()
    net = FusedActor(model, batchsize=nn_batch, dtype=torch.float16, cuda_graph=False)
    opts = dict(num_rollouts=rollouts, num_rollouts_per_batch=8, root_epsilon=0.25, root_alpha=0.03,
                nodes_per_game=nodes_per_game)
    host, dev = HostLoop(G, n, net, opts), DevLoop(G, n, net, opts)
    forms = {"host": host.move, "dev": dev.move}
    host.move()  # warm-up: every shape of every form
    dev.move()
    if graph:
        dev.capture()
        dev.replay()
        forms["graph"] = dev.replay
    secs = {k: [] for k in forms}
    for _ in range(rounds):  # alternate the forms
        for k, fn in forms.items():
            secs[k].append(timed(fn, moves))
    out = {"config": name, "G": G, "board": n, "tower": f"{blocks}x{dim}", "rollouts": rollouts, "moves_per_round": moves,
           "rounds": rounds, "card": card()}
    for k, s in secs.items():
        best = min(s)
        out[f"{k}_moves_per_s"] = round(moves / best, 2)
        out[f"{k}_game_moves_per_s"] = round(moves * G / best, 1)
        out[f"{k}_s_per_round"] = [round(x, 4) for x in s]
    if graph:
        out["graph_vs_host"] = round(out["graph_moves_per_s"] / out["host_moves_per_s"], 3)
    out["dev_vs_host"] = round(out["dev_moves_per_s"] / out["host_moves_per_s"], 3)
    print(json.dumps(out), flush=True)
    del host, dev, net, model
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--moves", type=int, default=10, help="moves per timed round (small configurations)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--big-moves", type=int, default=1, help="moves per timed round at the benchmark's configuration")
    ap.add_argument("--big-rounds", type=int, default=1)
    ap.add_argument("--configs", default="small,big", help="small (the two 6x64 configurations), big (the "
                    "benchmark's; about 95 s per move and form on an H100)")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("search_graph_bench needs a CUDA device")
    print(f"[search_graph_bench] {card()}", flush=True)
    which, res = a.configs.split(","), []
    if "small" in which:
        res += [run("9x9 6x64", 1024, 9, 6, 64, 64, 8192, a.moves, a.rounds, True),
                run("19x19 6x64", 512, 19, 6, 64, 64, 4096, a.moves, a.rounds, True)]
    if "big" in which:
        res.append(run("bench 20x256", 4096, 19, 20, 256, 800, 1024, a.big_moves, a.big_rounds, False, 900))
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(r) for r in res) + "\n")


if __name__ == "__main__":
    main()
