#!/usr/bin/env python
"""Self-play client on the GPU engine -- the counterpart of the reference's
``scripts/elfgames/go/selfplay.py`` / ``start_selfplay.sh`` for this path.

One process per GPU (``torchrun --nproc-per-node N scripts/selfplay.py ...``): every rank plays
its own ``--games`` games; rank 0's network weights are broadcast over NCCL once (the only
collective), game records in the reference's JSON wire format go to ``--records-out.<rank>``.

    python scripts/selfplay.py --games 4096 --rollouts 800 --blocks 20 --dim 256 --finish 4096
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=4096, help="concurrent games on this GPU")
    ap.add_argument("--board", type=int, default=19, choices=[9, 19])
    ap.add_argument("--rollouts", type=int, default=800)          # --mcts_rollout_per_thread
    ap.add_argument("--per-batch", type=int, default=8)           # --mcts_rollout_per_batch
    ap.add_argument("--puct", type=float, default=1.5)            # --mcts_puct
    ap.add_argument("--virtual-loss", type=int, default=1)        # --mcts_virtual_loss
    ap.add_argument("--root-epsilon", type=float, default=0.0)    # --mcts_epsilon
    ap.add_argument("--root-alpha", type=float, default=0.03)     # --mcts_alpha
    ap.add_argument("--policy-distri-cutoff", type=int, default=20)
    ap.add_argument("--resign-thres", type=float, default=0.05)
    ap.add_argument("--never-resign-ratio", type=float, default=0.1)
    ap.add_argument("--komi", type=float, default=7.5)
    ap.add_argument("--blocks", type=int, default=20)
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--nn-batch", type=int, default=256)
    ap.add_argument("--load", default=None, help="state_dict saved by the reference trainer (save-<step>.bin) or torch.save")
    ap.add_argument("--finish", type=int, default=0, help="stop after this many finished games on this rank (0 = run --moves)")
    ap.add_argument("--moves", type=int, default=10, help="number of move-steps when --finish is 0")
    ap.add_argument("--records-out", default=None)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--use-df-feature", action="store_true",
                    help="a DarkForest-plane network (GameOptions::use_df_feature): 25 input planes, float32 leaf batches")
    args = ap.parse_args()

    import torch

    import elf_b200
    from elf_b200.model import FusedActor, PolicyValueNet, broadcast_weights, load_reference_state_dict

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        import torch.distributed as dist

        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    torch.manual_seed(args.seed)
    planes = 25 if args.use_df_feature else 18
    net = PolicyValueNet(args.board, num_planes=planes, num_block=args.blocks, dim=args.dim).to(f"cuda:{local}")
    if args.load and rank == 0:
        sd = torch.load(args.load, map_location=f"cuda:{local}")
        missing, unexpected = load_reference_state_dict(net, sd)
        print(f"[selfplay] loaded {args.load}: {len(missing)} missing / {len(unexpected)} unexpected keys", file=sys.stderr)
    broadcast_weights(net)
    # frozen-network inference engine: BatchNorm folded, fused cuDNN epilogues, a full NN batch as a CUDA graph;
    # the search hands it the leaf batch as fp16 channels-last (no cast/permute pass); the DarkForest planes come
    # as float32 "s" and are converted in one pass into 32 padded channels
    actor = FusedActor(net.eval(), batchsize=args.nn_batch, dtype=torch.float16, cuda_graph=True,
                       cpad=32 if args.use_df_feature else 24)
    sp = elf_b200.selfplay.SelfPlay(
        actor, num_games=args.games, board_size=args.board, device=local,
        policy_distri_cutoff=args.policy_distri_cutoff, resign_thres=args.resign_thres,
        never_resign_ratio=args.never_resign_ratio, komi=args.komi, seed=args.seed + rank,
        record_games=args.records_out is not None, num_rollouts=args.rollouts,
        num_rollouts_per_batch=args.per_batch, c_puct=args.puct, virtual_loss=args.virtual_loss,
        persistent_tree=1, root_epsilon=args.root_epsilon, root_alpha=args.root_alpha, rotation_flip=1,
        **({"use_df_feature": True} if args.use_df_feature else {"feature_format": "f16"}))
    t0 = time.perf_counter()
    steps = 0
    while (sp.games_finished < args.finish) if args.finish > 0 else (steps < args.moves):
        sp.step()
        steps += 1
        if rank == 0 and steps % 10 == 0:
            dt = time.perf_counter() - t0
            bw = sum(1 for fv, _, _ in sp.results if fv > 0)
            print(f"[selfplay] step {steps}: {sp.moves_played} moves ({sp.moves_played / dt:.1f}/s), "
                  f"{sp.games_finished} games finished, black wins {bw}", file=sys.stderr, flush=True)
    dt = time.perf_counter() - t0
    if args.records_out:
        with open(f"{args.records_out}.{rank}", "w") as f:
            json.dump(sp.records, f)
    print(json.dumps({"rank": rank, "moves": sp.moves_played, "games_finished": sp.games_finished,
                      "seconds": dt, "moves_per_s": sp.moves_played / dt, "nn_positions": actor.num_positions,
                      "tree_prunes": int(sp.mcts.errors()[3]), "pool_overflows": int(sp.mcts.errors()[1])}), flush=True)
    sp.close()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
