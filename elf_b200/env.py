"""GoEnv: a batch of Go games on the GPU that a caller with its own policy drives from device tensors.

One ``step`` is one launch of ``elfb200_env_step`` (include/elfb200.h): every game plays its action, games
that end are scored (``GoState::evaluate``, black's view) and restarted from the empty board, and the
legal mask and info words of the positions now to move are written, plus the AGZ planes when asked for.
Nothing goes through the host, so ``policy -> step`` can be captured in a CUDA graph::

    env = GoEnv.create(4096, board_size=19, features="f16")
    obs = env.reset()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(64):
            obs = env.step(policy(obs["planes"], obs["legal"]))
    g.replay()

The observation tensors are allocated once, so their addresses stay fixed across steps and replays.
"""
import torch

from . import lib as _l
from .board import GoBatch

_FORMATS = {"f32": _l.FEAT_F32_NCHW, "f16": _l.FEAT_F16_NHWC, "bf16": _l.FEAT_BF16_NHWC, "df": _l.FEAT_DF_F32_NCHW}


def random_legal_actions(legal, counter, seed=0):
    """A seeded uniform random policy in tensor ops, for benchmarks and tests: per game a move drawn
    uniformly from the legal non-pass moves of ``legal`` (bool [G, N*N+1]), pass only when no other move
    is legal.  The random state is ``counter``, an int64 [1] tensor on the same device that this call
    advances by one, so the policy can be captured in a CUDA graph and replays a fresh draw each time.
    Returns int32 [G]."""
    G, A = legal.shape
    M = 0xFFFFFFFF
    x = torch.arange(G * (A - 1), device=legal.device, dtype=torch.int64).view(G, A - 1)
    x = (x + counter * 0x9E3779B1 + int(seed) * 0x85EBCA77) & M  # every product stays below 2^63
    for _ in range(2):  # 32-bit integer hash (xor-shift-multiply)
        x = (((x >> 16) ^ x) * 0x45D9F3B) & M
    x = (x >> 16) ^ x
    moves = legal[:, : A - 1]
    pick = torch.where(moves, x, -1).argmax(1)
    counter.add_(1)
    return torch.where(moves.any(1), pick, A - 1).to(torch.int32)


class GoEnv:
    """``board``: a :class:`GoBatch` (or an object with its ``_lib`` / ``_ctx`` / ``num_games`` /
    ``board_size`` / ``device`` / ``stream`` attributes).  ``features``: None (no planes), ``"f32"``
    (float32 ``[G,18,N,N]``), ``"f16"`` / ``"bf16"`` (``[G,N,N,cpad]`` channels-last) or ``"df"`` (the 25
    DarkForest planes of ``GameOptions::use_df_feature``, float32 ``[G,25,N,N]``).  ``device``: where
    the observation tensors live, by default the board's CUDA device; a board whose kernels run on the host
    (the SIMT emulator build used by the tests) takes ``"cpu"``, and then no stream work is done.

    Observation dict (the same tensors after every call): ``ok`` uint8 [G] (the move was accepted),
    ``done`` uint8 [G] (the game ended on this step and was restarted), ``value`` float32 [G] (its
    ``GoState::evaluate(komi)`` from black's point of view, 0 where not done), ``legal`` bool [G,N*N+1],
    ``info`` int32 [G,12] (as ``GoBatch.info``) and ``planes`` (None without features)."""

    def __init__(self, board, komi=7.5, features=None, cpad=24, device=None):
        if features is not None and features not in _FORMATS:
            raise ValueError("features must be None, 'f32', 'f16', 'bf16' or 'df'")
        self.board = board
        self._lib, self._ctx = board._lib, board._ctx
        G, n = board.num_games, board.board_size
        self.num_games, self.board_size, self.num_actions = G, n, n * n + 1
        self.komi = float(komi)
        self.device = torch.device("cuda", board.device) if device is None else torch.device(device)
        self._cuda = self.device.type == "cuda"
        dev = self.device
        self.ok = torch.zeros(G, dtype=torch.uint8, device=dev)
        self.done = torch.zeros(G, dtype=torch.uint8, device=dev)
        self.value = torch.zeros(G, dtype=torch.float32, device=dev)
        self._legal = torch.zeros((G, n * n + 1), dtype=torch.uint8, device=dev)
        self.legal = self._legal.view(torch.bool)
        self.info = torch.zeros((G, _l.INFO_FIELDS), dtype=torch.int32, device=dev)
        self.features, self.cpad = features, int(cpad)
        self._fmt = _FORMATS.get(features)
        if features is None:
            self.planes = None
        elif features in ("f32", "df"):
            self.planes = torch.zeros((G, 18 if features == "f32" else 25, n, n), dtype=torch.float32, device=dev)
        else:
            dt = torch.float16 if features == "f16" else torch.bfloat16
            self.planes = torch.zeros((G, n, n, self.cpad), dtype=dt, device=dev)
        self.obs = {"ok": self.ok, "done": self.done, "value": self.value, "legal": self.legal, "info": self.info,
                    "planes": self.planes}
        if self._cuda:
            self._stream = torch.cuda.ExternalStream(board.stream, device=dev)
            self._ev_in, self._ev_out = torch.cuda.Event(), torch.cuda.Event()
        self._own_board = False

    @classmethod
    def create(cls, num_games, board_size=19, device=0, **kw):
        env = cls(GoBatch(num_games, board_size=board_size, device=device), **kw)
        env._own_board = True
        return env

    def close(self):
        if self._own_board:
            self.board.close()

    def _check(self, t, dtype, shape, name):
        if t.device != self.device or t.dtype not in dtype or tuple(t.shape) != shape or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous {'/'.join(map(str, dtype))} tensor of shape {shape} on "
                             f"{self.device}")

    def _enqueue(self, call, d4):
        """``call`` and the planes on the context stream, ordered after the caller's current stream and
        before its next work: events only, no host synchronisation"""
        if self._cuda:
            cur = torch.cuda.current_stream(self.device)
            self._ev_in.record(cur)
            self._stream.wait_event(self._ev_in)
        call()
        if self.planes is not None:
            d4p = None
            if d4 is not None:
                self._check(d4, (torch.int32,), (self.num_games,), "d4")
                d4p = d4.data_ptr()
            _l.check(self._lib, self._lib.elfb200_features_dev_ex(self._ctx, d4p, self.planes.data_ptr(), self._fmt,
                                                                  self.cpad))
        if self._cuda:
            self._ev_out.record(self._stream)
            cur.wait_event(self._ev_out)
        return self.obs

    def step(self, actions, d4=None):
        """one ply: ``actions`` int32 [G] on the env's device (x*N+y, N*N = pass, < 0 = leave the game as
        it is); ``d4``: optional int32 [G] D4 codes of the planes.  Returns the observation dict."""
        self._check(actions, (torch.int32,), (self.num_games,), "actions")
        L, c = self._lib, self._ctx
        return self._enqueue(lambda: _l.check(L, L.elfb200_env_step(
            c, actions.data_ptr(), self.komi, self.ok.data_ptr(), self.done.data_ptr(), self.value.data_ptr(),
            self._legal.data_ptr(), self.info.data_ptr())), d4)

    def reset(self, mask=None, d4=None):
        """restart every game (``mask`` None) or the games where the uint8 / bool [G] device tensor ``mask`` is
        set, e.g. games the caller's policy resigned (the caller scores those itself); ``ok``, ``done`` and
        ``value`` are cleared.  Returns the observation of the positions now to move."""
        mptr = None
        if mask is not None:
            self._check(mask, (torch.uint8, torch.bool), (self.num_games,), "mask")
            mask = mask.view(torch.uint8)
            mptr = mask.data_ptr()
        self.ok.zero_()
        self.done.zero_()
        self.value.zero_()
        L, c = self._lib, self._ctx

        def call():
            _l.check(L, L.elfb200_reset_dev(c, mptr))
            _l.check(L, L.elfb200_observe_dev(c, self._legal.data_ptr(), self.info.data_ptr()))

        return self._enqueue(call, d4)

    def load(self, src, index, d4=None):
        """copy positions into this env's games: game i becomes a copy of game ``index[i]`` of ``src`` (a
        :class:`GoBatch` or a ``GoEnv`` of the same board size on the same device) for ``index[i]`` in
        [0, src.num_games); any other value leaves game i as it is.  ``index``: int32 [G] on the env's device,
        e.g. ``torch.where(done, pick, -1)`` to restart finished games from a pool of positions.  ``ok``,
        ``done`` and ``value`` of the loaded games are cleared, as ``reset`` clears them.  Returns the
        observation of every game, as ``observe``."""
        board = src.board if isinstance(src, GoEnv) else src
        self._check(index, (torch.int32,), (self.num_games,), "index")
        loaded = (index >= 0) & (index < board.num_games)
        for t in (self.ok, self.done, self.value):
            t.masked_fill_(loaded, 0)
        self.board.gather(board, index if self._cuda else index.numpy())
        return self.observe(d4)

    def observe(self, d4=None):
        """the observation of the stored positions without playing, e.g. after ``board.place_handicap``"""
        L, c = self._lib, self._ctx
        return self._enqueue(lambda: _l.check(L, L.elfb200_observe_dev(c, self._legal.data_ptr(), self.info.data_ptr())),
                             d4)
