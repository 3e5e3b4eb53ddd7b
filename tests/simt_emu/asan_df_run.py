"""Memcheck of the DarkForest leaf writer without a GPU: the emulator build under AddressSanitizer (as
asan_run.py), driving k_leaf_features_df with a node pool small enough to overflow, random D4 codes, a
persistent tree over several moves (the parent chains k_leaf_features_df walks span moves) and the
board batch's DF format.

    python tests/simt_emu/asan_df_run.py            (re-executes itself with libasan preloaded)

TEST INFRASTRUCTURE ONLY."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def main():
    if os.environ.get("SIMT_EMU_ASAN_CHILD") != "1":
        asan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
        env = dict(os.environ, LD_PRELOAD=os.path.realpath(asan), SIMT_EMU_ASAN_CHILD="1",
                   ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0")
        sys.exit(subprocess.call([sys.executable, os.path.abspath(__file__)], env=env))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    import numpy as np
    import torch

    import build
    from elf_b200 import lib as _l
    from tests import emu as E
    from tests.df_search import callback

    E._lib = _l.load_library(build.build(asan=True))
    for n, G in ((9, 5), (19, 2)):
        gb = E.emu_batch(G, n)
        rng = np.random.default_rng(n)
        for _ in range(12):
            legal = gb.legal_mask()[:, :-1]
            gb.forward(np.array([int(rng.choice(np.flatnonzero(lg))) for lg in legal], np.int32))
        out = np.zeros((G, 25, n, n), np.float32)
        _l.check(E._lib, E._lib.elfb200_features_dev_ex(gb._ctx, None, out.ctypes.data, _l.FEAT_DF_F32_NCHW, 0))
        # R + 2 nodes per game: the pool overflows during the first move and the reused trees are pruned later
        mc = E.EmuSearch(gb, rotation_flip=1, num_rollouts=48, num_rollouts_per_batch=8, persistent_tree=1,
                         nodes_per_game=50)
        mc._fmt = _l.FEAT_DF_F32_NCHW
        mc.feat = torch.zeros((mc.max_leaves, 25, n, n), dtype=torch.float32)

        def net(batch):
            pi, v = callback(batch["s"].numpy())
            return {"pi": torch.from_numpy(pi), "V": torch.from_numpy(v)}

        for _ in range(6):
            mc.search(net)
            a, _v = mc.choose(0, 0.0)
            gb.forward(a)
            mc.advance(a)
        print(f"[asan df] {n}x{n}: errors {mc.errors().tolist()}", flush=True)
        mc.close()
        gb.close()
    print("[asan df] clean", flush=True)


if __name__ == "__main__":
    main()
