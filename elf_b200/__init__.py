"""elf_b200 -- H100-native (sm_90a) replacement for ELF OpenGo's data-parallel hot path.

Host-side mirror of the reference interface for that path:

* :class:`elf_b200.board.GoBatch`   -- a batch of ``GoState`` objects living in GPU memory
  (reference ``src_cpp/elfgames/go/base/go_state.h:95-228``).
* :class:`elf_b200.mcts.MctsBatch`  -- the batched tree search (``MCTSGoAI`` for G games).
* :class:`elf_b200.env.GoEnv`       -- the batch as an environment stepped, scored, restarted and observed
  from device tensors, for a caller that runs its own policy on the GPU.
* :mod:`elf_b200.selfplay` / :mod:`elf_b200.online` / :mod:`elf_b200.console` -- the self-play and
  online (GTP) game loops of ``GoGameSelfPlay``; :mod:`elf_b200.compat` -- the pybind surface the
  reference's Python scripts call; :mod:`elf_b200.sgf`, :mod:`elf_b200.record` -- SGF / record formats.
* :mod:`elf_b200.lib`               -- ctypes binding of the C ABI declared in ``include/elfb200.h``.

The CUDA library is mandatory: importing :mod:`elf_b200.lib` without ``libelfb200.so`` raises,
and every call fails without a CUDA device.  There is no CPU fallback.
"""
from .lib import ElfB200Error, load_library  # noqa: F401
from .board import GoBatch  # noqa: F401
from .mcts import MctsBatch  # noqa: F401
from .env import GoEnv  # noqa: F401
from . import selfplay  # noqa: F401

__all__ = ["GoBatch", "MctsBatch", "GoEnv", "ElfB200Error", "load_library"]
