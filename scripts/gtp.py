#!/usr/bin/env python
"""GTP engine on the GPU search -- the counterpart of the reference's
``scripts/elfgames/go/df_console.py`` / ``gtp.sh`` (one game, MCTS per ``genmove``).

    python scripts/gtp.py --load pretrained-go-19x19-v2.bin --rollouts 1600 < commands.gtp

The whole move search (select / leaf features / expand / backup) runs in CUDA for the single game;
the network is evaluated on ``--per-batch`` leaves per wave.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--board", type=int, default=19, choices=[9, 19])
    ap.add_argument("--rollouts", type=int, default=1600)         # --mcts_rollout_per_thread x --mcts_threads
    ap.add_argument("--per-batch", type=int, default=16)          # --mcts_rollout_per_batch: leaves per network call
    ap.add_argument("--puct", type=float, default=1.5)
    ap.add_argument("--virtual-loss", type=int, default=1)
    ap.add_argument("--komi", type=float, default=7.5)
    ap.add_argument("--resign-thres", type=float, default=0.05)
    ap.add_argument("--blocks", type=int, default=20)
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--load", default=None, help="state_dict saved by the reference trainer or torch.save")
    ap.add_argument("--preload-sgf", default=None)
    ap.add_argument("--preload-sgf-move-to", type=int, default=-1)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--use-df-feature", action="store_true",
                    help="a DarkForest-plane network (GameOptions::use_df_feature): 25 input planes")
    ap.add_argument("--pass-alive", action="store_true",
                    help="final_status_list: pass-alive groups are never dead, opponent stones in their area always are")
    args = ap.parse_args()

    import torch

    from elf_b200.console import GtpConsole
    from elf_b200.model import Actor, PolicyValueNet, load_reference_state_dict
    from elf_b200.online import OnlineGame

    torch.cuda.set_device(args.device)
    net = PolicyValueNet(args.board, num_planes=25 if args.use_df_feature else 18, num_block=args.blocks,
                         dim=args.dim).to(f"cuda:{args.device}")
    if args.load:
        sd = torch.load(args.load, map_location=f"cuda:{args.device}")
        missing, unexpected = load_reference_state_dict(net, sd)
        print(f"[gtp] loaded {args.load}: {len(missing)} missing / {len(unexpected)} unexpected keys", file=sys.stderr)
    else:
        print("[gtp] no --load given: playing with random weights", file=sys.stderr)
    actor = Actor(net, batchsize=args.per_batch)
    game = OnlineGame.create(
        board_size=args.board, device=args.device, komi=args.komi, resign_thres=args.resign_thres,
        preload_sgf=args.preload_sgf, preload_sgf_move_to=args.preload_sgf_move_to, num_rollouts=args.rollouts,
        num_rollouts_per_batch=args.per_batch, c_puct=args.puct, virtual_loss=args.virtual_loss, persistent_tree=1,
        rotation_flip=1, use_df_feature=args.use_df_feature)
    console = GtpConsole(game, actor)
    console.final_status_pass_alive = args.pass_alive
    console.run()


if __name__ == "__main__":
    main()
