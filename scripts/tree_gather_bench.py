#!/usr/bin/env python
"""Copying search trees between handles (elfb200_mcts_gather_dev, k_gather_trees) on the H100.  Prints one JSON
line with the card's name and power limit, read in the same run.

Workload: 2048 19x19 games, 16 seeded random opening plies, three searched moves at 800 rollouts (waves of 8,
persistent trees, tests/planenet.py's plane-digest net, the most visited move played and advanced into); then
the trees are copied into a second handle of 2048 games with a random permutation.

  copy_us      device events around `--reps` back-to-back elfb200_mcts_gather_dev calls on the destination
               stream (after `--warmup` calls), per call
  nodes, edges in-use nodes and stored edges of the visited nodes over all source trees (elfb200_mcts_tree_usage,
               read back once): what the copy must move
  moved_MB     every copied record read once and written once: per in-use node the pos and sa rows (2 x 8 N B),
               hash (8 B), meta (16 B) and header (32 B); per stored edge 16 B of estat and 4 B of elink; the
               free stack (2 B per free slot); plus a 1-byte status store per free slot
  hbm_frac     moved bytes / copy time over the H100 SXM data sheet's 3.35 TB/s"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elf_b200 import lib as _l  # noqa: E402

PEAK_GBS = 3350.0  # H100 SXM data sheet (HBM3)
DEV = torch.device("cuda", 0)


def gpu_name_and_power():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in out.split(","))
    return name, power


def moved_bytes(n, C, nodes, edges):
    free = C * len(nodes) - int(nodes.sum())
    per_node = 2 * 8 * n + 8 + 16 + 32
    return 2 * (int(nodes.sum()) * per_node + int(edges.sum()) * 20 + 2 * free) + free


def main():
    import elf_b200
    from tests import planenet
    from tests.search_scale import OPENING_PLIES, random_opening

    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=2048)
    ap.add_argument("--board", type=int, default=19)
    ap.add_argument("--rollouts", type=int, default=800)
    ap.add_argument("--moves", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    n, G, R = args.board, args.games, args.rollouts
    opts = dict(num_rollouts=R, num_rollouts_per_batch=8, virtual_loss=1, persistent_tree=1, c_puct=1.5, rotation_flip=0)
    net = planenet.PlaneNet(n, "cuda", batchsize=0)
    src = elf_b200.GoBatch(G, board_size=n)
    random_opening([src], OPENING_PLIES, np.random.default_rng(1))
    sm = elf_b200.MctsBatch(src, **opts)
    for _ in range(args.moves):
        sm.search(net)
        a, _ = sm.choose(0, 0.0)
        src.forward(a)
        sm.advance(a)
    dst = elf_b200.GoBatch(G, board_size=n)
    dm = elf_b200.MctsBatch(dst, **opts)
    idx = torch.from_numpy(np.random.default_rng(2).permutation(G).astype(np.int32)).to(DEV)
    nodes, edges = sm.tree_usage()
    C = dm._lib.elfb200_mcts_nodes_per_game(dm._m)
    L = dm._lib
    st = torch.cuda.ExternalStream(dst.stream, device=DEV)
    for _ in range(args.warmup):
        _l.check(L, L.elfb200_mcts_gather_dev(dm._m, sm._m, idx.data_ptr()))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(args.reps):
        _l.check(L, L.elfb200_mcts_gather_dev(dm._m, sm._m, idx.data_ptr()))
    e1.record(st)
    e1.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / args.reps
    dn, de = dm.tree_usage()
    ix = idx.cpu().numpy()
    assert (dn == nodes[ix]).all() and (de == edges[ix]).all()
    moved = moved_bytes(n, C, nodes, edges)
    name, power = gpu_name_and_power()
    print(json.dumps({"gpu": name, "power_limit": power, "board": n, "games": G, "rollouts": R, "moves": args.moves,
                      "nodes_per_game": C, "mean_nodes": round(float(nodes.mean()), 1),
                      "mean_edges": round(float(edges.mean()), 1), "copy_us": round(us, 1),
                      "moved_MB": round(moved / 1e6, 1), "moved_GBs": round(moved / us / 1e3, 1),
                      "hbm_frac": round(moved / us / 1e3 / PEAK_GBS, 3), "reps": args.reps}), flush=True)
    for x in (sm, dm, src, dst):
        x.close()


if __name__ == "__main__":
    main()
