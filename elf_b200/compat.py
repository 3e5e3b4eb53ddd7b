"""compat -- the reference's Python-visible batching surface, served by the GPU engine.

The reference's scripts talk to C++ through three pybind objects (SURVEY.md 8b):

* ``GameContext(ContextOptions, GameOptions)`` with ``.ctx()`` and ``.getParams()``
  (``src_cpp/elfgames/go/train/Pybind.cc:22-62``, ``inference/Pybind.cc:22-43``);
* ``elf::Context`` with ``createSharedMemOptions / allocateSharedMem / start / wait / step / stop /
  version`` (``src_cpp/elf/Pybind.cc:46-62``);
* ``SharedMem`` / ``AnyP`` through which ``GCWrapper`` (``src_py/elf/utils_elf.py:32-57,378-405``)
  learns each field's name / element type / shape and registers the memory it allocated
  (``AnyP.set(ptr, byte_strides)``, ``src_cpp/elf/base/extractor.h:302-305``).

This module re-creates exactly that surface in Python on top of the batched GPU search, so the
unmodified ``GCWrapper.run()`` loop -- ``smem = ctx.wait(); cb(batch) -> reply; ctx.step()`` -- and
the unmodified rlpytorch ``Evaluator.actor`` callback drive it:

* ``wait()`` advances the engine to the next chunk (<= the label's batchsize) of MCTS leaves that
  need the network, writes their feature planes into the tensor registered for ``"s"`` and returns
  the label's ``SharedMem`` with ``effective_batchsize()`` set;
* ``step()`` reads ``"pi"`` / ``"V"`` back from the registered reply tensors; when the last chunk
  of a wave has been answered the engine expands, backs up and carries on (next wave, or move
  selection + ``GoState::forward`` + tree advance for every game).

Registered memory may be pinned host memory (the reference's ``Allocator``; features are copied
device->host, replies host->device) or CUDA memory (fast mode: device-to-device copies only).

There are no game threads: the search of all games runs on the GPU between two ``wait()`` calls.
"""
import ctypes

import numpy as np

_TYPES = {  # GoFeature::registerExtractor element types (common/game_feature.h:159-206)
    "float": (np.float32, "float"),
    "int64_t": (np.int64, "int64_t"),
    "int32_t": (np.int32, "int32_t"),
}


class Size:
    def __init__(self, dims):
        self._d = [int(x) for x in dims]

    def vec(self):
        return list(self._d)


class FieldInfo:
    def __init__(self, name, type_name, dims):
        self._n, self._t, self._s = name, type_name, Size(dims)

    def name(self):
        return self._n

    def type_name(self):
        return self._t

    def sz(self):
        return self._s


class AnyP:
    """One field of one SharedMem: shape/type description + the caller's memory (AnyP, extractor.h:280-360)."""

    def __init__(self, name, type_name, dims):
        self._field = FieldInfo(name, type_name, dims)
        self.ptr = 0
        self.strides = None
        self._view = None

    def field(self):
        return self._field

    def set(self, ptr, strides):
        self.ptr = int(ptr)
        self.strides = [int(s) for s in strides]
        self._view = None

    setAddress = set

    def view(self):
        """torch tensor aliasing the registered memory (host or device)"""
        import torch

        if self._view is not None:
            return self._view
        if not self.ptr:
            raise RuntimeError(f"field {self._field.name()} has no memory registered (AnyP.set was not called)")
        dims = self._field.sz().vec()
        npdt = _TYPES[self._field.type_name()][0]
        item = np.dtype(npdt).itemsize
        attr = None
        try:
            try:
                from cuda.bindings import runtime as cudart  # cuda-python >= 12.8
            except Exception:
                from cuda import cudart

            err, a = cudart.cudaPointerGetAttributes(self.ptr)
            if int(err) == 0:
                attr = int(a.type)
        except Exception:
            attr = None
        is_dev = attr == 2  # cudaMemoryTypeDevice
        if is_dev:
            class _CAI:  # __cuda_array_interface__ holder
                pass

            o = _CAI()
            o.__cuda_array_interface__ = {
                "shape": tuple(dims), "typestr": np.dtype(npdt).str, "data": (self.ptr, False), "version": 3,
                "strides": tuple(self.strides),
            }
            self._view = torch.as_tensor(o, device="cuda")
        else:
            nbytes = sum((d - 1) * s for d, s in zip(dims, self.strides)) + item
            buf = (ctypes.c_char * nbytes).from_address(self.ptr)
            arr = np.ndarray(shape=tuple(dims), dtype=npdt, buffer=buf, strides=tuple(self.strides))
            self._view = torch.from_numpy(arr)
        return self._view


class SharedMemOptions:
    def __init__(self, idx, label, batchsize):
        self._idx, self._label, self._bs, self._timeout = idx, label, int(batchsize), 0

    def idx(self):
        return self._idx

    def label(self):
        return self._label

    def batchsize(self):
        return self._bs

    def setTimeout(self, usec):
        self._timeout = int(usec)

    def info(self):
        return f"SMem[{self._label}], idx: {self._idx}, batchsize: {self._bs}"


class SharedMem:
    def __init__(self, opts, fields):
        self._opts = opts
        self._fields = fields
        self._eff = 0

    def __getitem__(self, key):
        return self._fields[key]

    def getSharedMemOptions(self):
        return self._opts

    def effective_batchsize(self):
        return self._eff

    def info(self):
        return self._opts.info()


class ReplyStatus:
    SUCCESS, FAILED, UNKNOWN = 0, 1, 2


class Context:
    """elf::Context (src_cpp/elf/base/context.h:110-394) as seen from Python."""

    def __init__(self, engine, batchsize):
        self._engine = engine
        self._batchsize = int(batchsize)  # co.batchsize: every field's leading extent
        self._smems = []
        self._by_label = {}
        self._rr = {}
        self._cur = None
        self._started = False
        self._stopped = False

    def version(self):
        return "elf_b200-compat"

    def createSharedMemOptions(self, name, batchsize):
        return SharedMemOptions(-1, name, batchsize)

    def _field_dims(self, key):
        n, a = self._engine.board_size, self._engine.num_action
        bs = self._batchsize
        k = int(getattr(self._engine, "num_future_actions", 1))
        planes = int(getattr(self._engine, "num_planes", 18))
        table = {  # GoFeature::registerExtractor, common/game_feature.h:159-183
            "s": ("float", [bs, planes, n, n]), "pi": ("float", [bs, a]), "V": ("float", [bs]),
            "a": ("int64_t", [bs]), "rv": ("int64_t", [bs]),
            "black_ver": ("int64_t", [bs]), "white_ver": ("int64_t", [bs]), "selfplay_ver": ("int64_t", [bs]),
            "offline_a": ("int64_t", [bs, k]), "winner": ("float", [bs]), "predicted_value": ("float", [bs]),
            "mcts_scores": ("float", [bs, a]), "move_idx": ("int32_t", [bs]), "aug_code": ("int32_t", [bs]),
            "num_move": ("int32_t", [bs]),
        }
        if key not in table:
            raise KeyError(f"field '{key}' is not provided by the elf_b200 engine")
        return table[key]

    def allocateSharedMem(self, opts, keys):
        o = SharedMemOptions(len(self._smems), opts.label(), opts.batchsize())
        o.setTimeout(opts._timeout)
        fields = {}
        for k in keys:
            t, dims = self._field_dims(k)
            fields[k] = AnyP(k, t, dims)
        sm = SharedMem(o, fields)
        self._smems.append(sm)
        self._by_label.setdefault(o.label(), []).append(sm)
        return sm

    def start(self):
        self._started = True
        self._engine.start()

    def stop(self):
        self._stopped = True
        self._engine.stop()

    def _next_smem(self, label):
        sms = self._by_label[label]
        i = self._rr.get(label, 0)
        self._rr[label] = (i + 1) % len(sms)  # num_recv SharedMems are used round-robin
        return sms[i]

    def wait(self, timeout_usec=0):
        if not self._started or self._stopped:
            raise RuntimeError("Context.wait() outside start()/stop()")
        # game_start / game_end notifications (batchsize 1, game.py:398-405) come first
        poll = getattr(self._engine, "poll_event", None)
        nl = getattr(self._engine, "next_label", None)
        while True:
            while poll is not None:
                ev = poll()
                if ev is None:
                    break
                label, fields = ev
                if label not in self._by_label:
                    continue  # the script did not ask for this label
                sm = self._next_smem(label)
                for k, val in fields.items():
                    if k in sm._fields:
                        sm[k].view()[:1] = val
                sm._eff = 1
                self._cur = sm
                return sm
            label = nl() if nl is not None else "actor_black"  # which AI's leaves come next
            if label is not None:
                break  # (None: the engine queued a notification that has to go out first)
        sms = self._by_label.get(label)
        if not sms:
            raise RuntimeError(f"no SharedMem allocated for label '{label}'")
        sm = self._next_smem(label)
        nf = getattr(self._engine, "next_fields", None)
        if nf is not None:  # engines that fill several input fields (the `train` label)
            n, fields = nf(sm.getSharedMemOptions().batchsize())
            for k, val in fields.items():
                if k in sm._fields:
                    sm[k].view()[:n].copy_(val, non_blocking=False)
        else:
            n, feats = self._engine.next_batch(sm.getSharedMemOptions().batchsize())
            dst = sm["s"].view()
            dst[:n].copy_(feats, non_blocking=False)
        sm._eff = int(n)
        self._cur = sm
        return sm

    def step(self, status=ReplyStatus.SUCCESS):
        sm = self._cur
        if sm is None:
            raise RuntimeError("Context.step() without a pending wait()")
        if sm.getSharedMemOptions().label() in ("game_start", "game_end"):
            self._cur = None  # notifications carry no reply
            return
        if sm.getSharedMemOptions().label() in ("train", "train_ctrl"):
            self._cur = None  # reply=None labels (game.py:407-418)
            return
        if sm.getSharedMemOptions().label() == "human_actor":
            # GoFeature::ReplyAction (common/game_feature.h:50-66): only "a" is consumed
            self._engine.reply_action(int(sm["a"].view().reshape(-1)[0]))
            self._cur = None
            return
        n = sm._eff
        pi = sm["pi"].view()[:n]
        v = sm["V"].view()[:n]
        self._engine.reply(pi, v)
        self._cur = None


class WinRateStats:  # common/game_stats.h:21-68 as exposed to Python (selfplay.py:161-166)
    def __init__(self, black_wins, white_wins):
        self.black_wins = int(black_wins)
        self.white_wins = int(white_wins)
        self.total_games = self.black_wins + self.white_wins


class _Client:
    def __init__(self, engine):
        self._e = engine

    def setRequest(self, black_ver, white_ver, resign_thres, num_threads=-1):  # distri_client.h:318-331
        """Client::setRequest: a local MsgRequest {vers, black/white_resign_thres = thres,
        num_game_thread_used} handed to every game through the dispatcher"""
        sr = getattr(self._e, "set_request", None)
        if sr is not None:
            sr(int(black_ver), int(white_ver), float(resign_thres), int(num_threads))
        else:
            self._e.resign_thres = float(resign_thres)

    def getGameStats(self):
        return self

    def getWinRateStats(self):
        return self._e.win_stats()


class GameContext:
    """go.GameContext (train/game_context.h:37-85, inference/game_context.h:31) over an engine."""

    def __init__(self, engine, batchsize):
        self._engine = engine
        self._ctx = Context(engine, batchsize)

    def ctx(self):
        return self._ctx

    def getParams(self):  # GoFeature::getParams, common/game_feature.h:208-221
        n = self._engine.board_size
        df = int(getattr(self._engine, "num_planes", 18)) == 25  # GoFeature ctor, game_feature.h:22-33
        return {
            "num_action": n * n + 1, "board_size": n, "num_future_actions": int(getattr(self._engine, "num_future_actions", 1)),
            "num_planes": 25 if df else 18, "our_stone_plane": 7 if df else 0, "opponent_stone_plane": 8 if df else 1,
            "ACTION_SKIP": -100, "ACTION_PASS": -99, "ACTION_RESIGN": -98, "ACTION_CLEAR": -97,
        }

    def getClient(self):
        return _Client(self._engine)

    def getGame(self, game_idx):
        """GameContext::getGame (inference/game_context.h:59-66): the object console_lib.py asks for
        showBoard / getNextPlayer / getLastMove / getScore / getLastScore"""
        return self._engine.game_view(int(game_idx))


class SelfPlayEngine:
    """The engine behind compat.Context: SelfPlay's move loop cut at the network round trip."""

    def __init__(self, selfplay):
        self.sp = selfplay
        self.board_size = selfplay.N
        self.num_action = selfplay.N * selfplay.N + 1
        self.num_planes = 25 if getattr(selfplay, "use_df_feature", False) else 18
        self.resign_thres = selfplay.resign_thres
        import collections

        self._events = collections.deque()
        self._pending = None  # a request waiting for the next move boundary
        self.replies = []  # RestartReply names of the requests applied so far
        self._wave = None  # (features tensor [n,...], n, offset, pi buffer, v buffer)
        self._wave_idx = 0
        self._in_move = False
        self._info = None

    def start(self):
        pass

    def stop(self):
        pass

    def win_stats(self):
        r = self.sp.results
        return WinRateStats(sum(1 for fv, _, _ in r if fv > 0), sum(1 for fv, _, _ in r if fv <= 0))

    def set_request(self, black_ver, white_ver=-1, resign_thres=None, num_game_thread_used=-1, **ctrl):
        """a MsgRequest for every game (Client::setRequest locally, or the training server's reply
        relayed by the caller).  It takes effect between two moves -- the reference's game threads
        look at the dispatcher every 5th move (game_selfplay.cc:273-290), here all games do at the
        next move boundary.  ``ctrl``: white_resign_thres, never_resign_prob, player_swap, async_."""
        self._pending = dict(black_ver=black_ver, white_ver=white_ver, black_resign_thres=resign_thres,
                             num_game_thread_used=num_game_thread_used, **ctrl)

    def _apply_pending(self):
        if self._pending is None or self._in_move:
            return
        req, self._pending = self._pending, None
        reply = self.sp.set_request(**req)
        self.resign_thres = self.sp.resign_thres
        self.replies.append(reply)
        if reply in ("update_model", "update_model_async"):
            # DispatcherCallback::OnReply (dispatcher_callback.h:46-99): ONE game_start per actionable
            # request carries the versions to Python, which loads the models (selfplay.py:138-156)
            self._events.append(("game_start", {"black_ver": req["black_ver"], "white_ver": req["white_ver"]}))

    def poll_event(self):
        self._apply_pending()
        return self._events.popleft() if self._events else None

    def _phases(self, info):
        """[(search, label, active, waves or None, post or None)] for this move; with a policy-only
        colour (GameOptions::black/white_use_policy_network_only) the plan is SelfPlay.policy_only_plan's"""
        sp = self.sp
        self._chosen = None
        if any(getattr(sp, "policy_only", {}).values()):
            G = sp.G
            self._chosen = (np.full(G, -2, np.int32), np.zeros(G, np.float32))
            return [(mc, label, active, waves, post)
                    for mc, _, label, active, waves, post in sp.policy_only_plan(info, *self._chosen)]
        return [(mc, label, active, None, None) for mc, _, label, active in sp.phases(info)]

    def _begin_phase(self, i):
        mc, _, active, waves, _ = self._plan[i]
        # a policy-only phase (waves given) takes no root noise (TreeSearchT::runPolicyOnly)
        noise = getattr(mc, "set_root_noise_enabled", None)
        if noise is not None:
            noise(waves is None)
        try:
            mc.begin_move(active)
        finally:
            if noise is not None:
                noise(True)
        self._wave_idx = 0

    def _advance_until_leaves(self):
        import torch

        sp = self.sp
        while True:
            if not self._in_move:
                if self._pending is not None:
                    self._apply_pending()
                    if self._events:
                        return False  # game_start has to reach Python before the new models are asked
                if sp.idle is not None and sp.idle.all():
                    raise RuntimeError("every game is waiting for a request (black_ver < 0): nothing to evaluate")
                self._info = sp.gb.info()
                self._plan = self._phases(self._info)
                self._phase = 0
                self._res = []
                self._begin_phase(0)
                self._in_move = True
            mc, label, _, waves, post = self._plan[self._phase]
            if self._wave_idx >= (mc.waves_per_move if waves is None else waves):
                if post is not None:
                    post()
                self._phase += 1
                if self._phase == len(self._plan):
                    self._finish_move()
                else:
                    self._begin_phase(self._phase)
                continue
            s = mc.select()
            self._wave_idx += 1
            n = s.shape[0]
            if n == 0:
                mc.expand_backup(None, None)
                continue
            sp.gb.synchronize()
            dev = s.device
            self._wave = {"s": s, "n": n, "off": 0, "got": 0, "mc": mc, "label": label,
                          "pi": torch.empty((n, self.num_action), dtype=torch.float32, device=dev),
                          "v": torch.empty((n,), dtype=torch.float32, device=dev)}
            return True

    def _finish_move(self):
        sp = self.sp
        sp.resign_thres = self.resign_thres
        before = sp.games_finished
        if self._chosen is not None:
            sp._policy_only_moves = sp._po_colour & (self._chosen[0] >= 0)
        sp.finish_move(self._info, chosen=self._chosen)
        for _ in range(sp.games_finished - before):  # finish_game -> GameNotifier::OnGameEnd -> game_end
            self._events.append(("game_end", {}))
        self._in_move = False

    def next_label(self):
        """label of the next leaf batch, or None when a notification has to be delivered first"""
        if self._wave is None or self._wave["off"] >= self._wave["n"]:
            if self._wave is not None and self._wave["got"] < self._wave["n"]:
                raise RuntimeError("wait() called again before step() answered the previous batch")
            if not self._advance_until_leaves():
                self._wave = None
                return None
        return self._wave["label"]

    def next_batch(self, max_n):
        if self._wave is None or self._wave["off"] >= self._wave["n"]:
            if self._wave is not None and self._wave["got"] < self._wave["n"]:
                raise RuntimeError("wait() called again before step() answered the previous batch")
            self._advance_until_leaves()
        w = self._wave
        k = min(int(max_n), w["n"] - w["off"])
        feats = w["s"][w["off"]:w["off"] + k]
        w["last"] = (w["off"], k)
        w["off"] += k
        return k, feats

    def reply(self, pi, v):
        import torch

        w = self._wave
        off, k = w["last"]
        w["pi"][off:off + k].copy_(pi.to(torch.float32), non_blocking=False)
        w["v"][off:off + k].copy_(v.to(torch.float32).reshape(-1), non_blocking=False)
        w["got"] += k
        if w["got"] >= w["n"]:
            if w["pi"].is_cuda:
                torch.cuda.current_stream(w["pi"].device).synchronize()
            w["mc"].expand_backup(w["pi"], w["v"])


class OnlineEngine:
    """mode == "online" behind compat.Context (game.py:363-374: labels ``human_actor`` with
    batchsize 1 and ``actor_black`` with batchsize num_rollouts_per_batch).

    ``wait()`` returns the ``human_actor`` SharedMem (features of the current position) whenever the
    game waits for the operator; the reply's ``a`` is a board action or one of the special actions
    (ACTION_SKIP lets the AI move).  While the AI is searching, ``wait()`` hands out ``actor_black``
    batches of MCTS leaves exactly like the self-play engine."""

    def __init__(self, game):
        self.game = game
        self.board_size = game.N
        self.num_action = game.N * game.N + 1
        self.num_planes = 25 if getattr(game, "use_df_feature", False) else 18
        self._gen = None
        self._wave = None
        self.last_status = None

    @property
    def resign_thres(self):
        return self.game.resign_thres

    @resign_thres.setter
    def resign_thres(self, v):
        self.game.resign_thres = float(v)

    def start(self):
        pass

    def stop(self):
        pass

    def win_stats(self):
        r = self.game.finished
        return WinRateStats(sum(1 for fv, _, _ in r if fv > 0), sum(1 for fv, _, _ in r if fv <= 0))

    def poll_event(self):
        return None

    def game_view(self, idx):
        if idx != 0:
            raise IndexError("online mode has exactly one game")
        return self.game

    def next_label(self):
        return "actor_black" if self._gen is not None else "human_actor"

    def next_batch(self, max_n):
        import torch

        if self._gen is None:
            b = self.game.board
            return 1, torch.from_numpy(b.features_df() if self.num_planes == 25 else b.features())
        w = self._wave
        if w["off"] >= w["n"]:
            raise RuntimeError("wait() called again before step() answered the previous batch")
        k = min(int(max_n), w["n"] - w["off"])
        feats = w["s"][w["off"]:w["off"] + k]
        w["last"] = (w["off"], k)
        w["off"] += k
        return k, feats

    def _set_wave(self, s):
        import torch

        n = s.shape[0]
        self._wave = {"s": s, "n": n, "off": 0, "got": 0,
                      "pi": torch.empty((n, self.num_action), dtype=torch.float32, device=s.device),
                      "v": torch.empty((n,), dtype=torch.float32, device=s.device)}

    def reply_action(self, a):
        self.last_status = self.game.human(a)
        if self.last_status != "skip":
            return
        if int(self.game.info()[9]):  # nothing to search in a finished position
            self.game._finish_game("illegal")
            return
        self._gen = self.game.ai_search()
        try:
            self._set_wave(next(self._gen))
        except StopIteration:
            self._gen = None
            self.game.ai_finish()

    def reply(self, pi, v):
        import torch

        w = self._wave
        off, k = w["last"]
        w["pi"][off:off + k].copy_(pi.to(torch.float32), non_blocking=False)
        w["v"][off:off + k].copy_(v.to(torch.float32).reshape(-1), non_blocking=False)
        w["got"] += k
        if w["got"] < w["n"]:
            return
        if w["pi"].is_cuda:
            torch.cuda.current_stream(w["pi"].device).synchronize()
        try:
            self._set_wave(self._gen.send((w["pi"], w["v"])))
        except StopIteration:
            self._gen = None
            self._wave = None
            self.game.ai_finish()


class TrainEngine:
    """mode == "train" behind compat.Context: every ``wait()`` returns one ``train`` batch
    (game.py:407-413: input s, offline_a, winner, mcts_scores, move_idx, selfplay_ver; no reply) drawn
    from the replay records by ``elf_b200.replay.ReplayBatch`` (GoGameTrain::act for the batch)."""

    def __init__(self, replay_batch):
        self.rb = replay_batch
        self.board_size = replay_batch.N
        self.num_action = replay_batch.N * replay_batch.N + 1
        self.num_future_actions = replay_batch.K
        self.num_planes = int(getattr(replay_batch, "num_planes", 18))
        self.batches = 0

    def start(self):
        pass

    def stop(self):
        pass

    def win_stats(self):
        return WinRateStats(0, 0)

    def poll_event(self):
        return None

    def next_label(self):
        return "train"

    def next_fields(self, max_n):
        import torch

        if max_n < self.rb.B:
            raise RuntimeError(f"the train label's batchsize ({max_n}) is smaller than the replay batch ({self.rb.B})")
        out = self.rb.sample()
        self.batches += 1
        return self.rb.B, {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in out.items()}


# ---- option objects and GameContext(ContextOptions, GameOptions) ---------------------------------------
class _Bag:
    """attribute bag with the reference struct's field names and defaults (pybind REGISTER_PYBIND_FIELDS)"""

    _defaults = {}

    def __init__(self, **kw):
        for k, v in self._defaults.items():
            setattr(self, k, v() if callable(v) else v)
        for k, v in kw.items():
            if k not in self._defaults:
                raise AttributeError(f"{type(self).__name__} has no field '{k}'")
            setattr(self, k, v)

    def info(self):
        return "\n".join(f"{k}: {getattr(self, k)}" for k in self._defaults)


class SearchAlgoOptions(_Bag):  # elf/ai/tree_search/tree_search_options.h:23-27
    _defaults = dict(use_prior=True, c_puct=5.0, unexplored_q_zero=False, root_unexplored_q_zero=False)


class TSOptions(_Bag):  # tree_search_options.h:77-96
    _defaults = dict(max_num_moves=0, num_threads=16, num_rollouts_per_thread=100, num_rollouts_per_batch=8,
                     verbose=False, verbose_time=False, seed=0, persistent_tree=False, root_epsilon=0.0,
                     root_alpha=0.0, log_prefix="", pick_method="most_visited", alg_opt=SearchAlgoOptions,
                     virtual_loss=0)


class ContextOptions(_Bag):  # elf/legacy/python_options_utils_cpp.h:19-47
    _defaults = dict(num_games=1, batchsize=0, T=1, job_id="", mcts_options=TSOptions)

    def print(self):
        print(self.info())


class GameOptions(_Bag):  # elfgames/go/common/go_game_specific.h:20-128 (fields the engine or the scripts touch)
    _defaults = dict(
        seed=0, num_games_per_thread=-1, mode="selfplay", use_mcts=False, use_mcts_ai2=False,
        black_use_policy_network_only=False, white_use_policy_network_only=False, data_aug=-1,
        start_ratio_pre_moves=0.5, ratio_pre_moves=0.0, move_cutoff=-1, policy_distri_cutoff=20,
        policy_distri_training_for_all=False, resign_thres=0.05, resign_thres_lower_bound=1e-9,
        resign_thres_upper_bound=0.50, resign_prob_never=0.1, resign_target_fp_rate=0.05, resign_target_hist_size=2500,
        num_reset_ranking=5000, preload_sgf="", preload_sgf_move_to=-1, use_df_feature=False, q_min_size=10,
        q_max_size=1000, num_reader=50, komi=7.5, ply_pass_enabled=0, white_puct=-1.0, white_mcts_rollout_per_batch=-1,
        white_mcts_rollout_per_thread=-1, eval_num_games=400, eval_thres=0.55, client_max_delay_sec=1200,
        selfplay_init_num=5000, selfplay_update_num=1000, selfplay_async=False, following_pass=False,
        cheat_eval_new_model_wins_half=False, cheat_selfplay_random_result=False, keep_prev_selfplay=False,
        eval_num_threads=1, expected_num_clients=-1, list_files=list, server_addr="", server_id="", port=0,
        verbose=False, print_result=False, dump_record_prefix="", num_future_actions=1)


def search_kwargs(ts, rollouts_per_thread=None, per_batch=None, c_puct=None):
    """TSOptions -> elfb200_mcts_options.  The reference runs ``num_threads`` search threads of
    ``num_rollouts_per_thread`` rollouts each on one tree; the GPU search does the same total number
    of rollouts as one deterministic sequence of waves."""
    rpt = ts.num_rollouts_per_thread if not rollouts_per_thread or rollouts_per_thread <= 0 else rollouts_per_thread
    return dict(
        num_rollouts=int(max(1, ts.num_threads) * rpt),
        num_rollouts_per_batch=int(ts.num_rollouts_per_batch if not per_batch or per_batch <= 0 else per_batch),
        virtual_loss=int(ts.virtual_loss), persistent_tree=int(bool(ts.persistent_tree)),
        use_prior=int(bool(ts.alg_opt.use_prior)), c_puct=float(ts.alg_opt.c_puct if not c_puct or c_puct <= 0 else c_puct),
        unexplored_q_zero=int(bool(ts.alg_opt.unexplored_q_zero)),
        root_unexplored_q_zero=int(bool(ts.alg_opt.root_unexplored_q_zero)),
        root_epsilon=float(ts.root_epsilon), root_alpha=float(ts.root_alpha))


def game_context(co, opt, board_size=19, device=0, factories=None):
    """``go.GameContext(co, opt)`` (train/game_context.h:37-85, inference/game_context.h:31-66): build the
    engine the options describe and return the GameContext the scripts pump.

    ``co`` / ``opt``: ContextOptions / GameOptions -- these classes or the reference's pybind objects
    (only attributes are read).  ``opt.mode``: "selfplay" (SelfPlay + SelfPlayEngine), "online"
    (OnlineGame + OnlineEngine) or "train" / "offline_train" (ReplayBatch + TrainEngine; the caller
    feeds records with ``GC._engine.rb.add_records``).  ``board_size`` is a compile-time constant of
    the reference (BOARD9x9).  ``factories``: {"selfplay"|"online"|"replay": callable(**kwargs)} to
    substitute the constructors (tests)."""
    f = dict(factories or {})
    ts = co.mcts_options
    pick = str(getattr(ts, "pick_method", "most_visited"))
    if pick not in ("most_visited", "strongest_prior", "uniform_random"):
        # TreeSearchT::chooseAction throws std::range_error (tree_search.h:521-524), a ValueError in Python
        raise ValueError("MCTS Pick method unknown! " + pick)
    if pick != "most_visited":
        raise NotImplementedError(f"mcts_pick_method '{pick}': the device-side move choice ranks root edges by visits "
                                  "(the default, and what every shipped script uses)")
    common = search_kwargs(ts)
    common.update(komi=float(opt.komi), ply_pass_enabled=int(opt.ply_pass_enabled))
    if opt.mode == "selfplay":
        from .selfplay import SelfPlay

        for cheat in ("cheat_eval_new_model_wins_half", "cheat_selfplay_random_result"):
            if bool(getattr(opt, cheat, False)):
                # server-plumbing debug switches that replace a game's result by a coin flip
                # (GoStateExt::setFinalValue, go_state_ext.h:86-99): not part of the engine, refused loudly
                raise NotImplementedError(f"GameOptions::{cheat} is not supported by the elf_b200 engine")
        kw = dict(
            actor=None, num_games=int(co.num_games), board_size=board_size, device=device,
            policy_distri_cutoff=int(opt.policy_distri_cutoff), resign_thres=float(opt.resign_thres),
            never_resign_ratio=float(opt.resign_prob_never), move_cutoff=int(opt.move_cutoff),
            seed=int(opt.seed), record_games=True,
            black_use_policy_network_only=bool(opt.black_use_policy_network_only),
            white_use_policy_network_only=bool(opt.white_use_policy_network_only),
            policy_distri_training_for_all=bool(opt.policy_distri_training_for_all),
            num_games_per_thread=int(opt.num_games_per_thread),
            white_mcts_opts={k: v for k, v in search_kwargs(ts, opt.white_mcts_rollout_per_thread,
                                                             opt.white_mcts_rollout_per_batch, opt.white_puct).items()
                             if v != common.get(k)},
            **common)
        if int(opt.seed) != 0:
            # GameOptions::seed != 0: every game thread's generator starts from it (game_base.h:32-38) and
            # the reference's games are reproducible -- ours are then the same games (elf_b200.refstream)
            kw["rng"] = "reference"
        if bool(getattr(opt, "use_df_feature", False)):
            kw["use_df_feature"] = True
        sp = f.get("selfplay", SelfPlay)(**kw)
        return GameContext(SelfPlayEngine(sp), batchsize=int(co.batchsize))
    if opt.mode == "online":
        from .online import OnlineGame

        kw = dict(board_size=board_size, device=device, komi=float(opt.komi), resign_thres=float(opt.resign_thres),
                  policy_distri_cutoff=int(opt.policy_distri_cutoff), move_cutoff=int(opt.move_cutoff),
                  preload_sgf=opt.preload_sgf or None, preload_sgf_move_to=int(opt.preload_sgf_move_to),
                  following_pass=bool(opt.following_pass), seed=int(opt.seed), **{k: v for k, v in common.items() if k != "komi"})
        if bool(getattr(opt, "use_df_feature", False)):
            kw["use_df_feature"] = True
        game = f.get("online", OnlineGame.create)(**kw)
        return GameContext(OnlineEngine(game), batchsize=int(co.batchsize))
    if opt.mode in ("train", "offline_train"):
        from .replay import ReplayBatch

        kw = dict(num_states=int(co.batchsize), board_size=board_size, device=device,
                  num_future_actions=int(opt.num_future_actions), seed=int(opt.seed),
                  use_df_feature=bool(getattr(opt, "use_df_feature", False)))
        rb = f.get("replay", ReplayBatch)(**kw)
        return GameContext(TrainEngine(rb), batchsize=int(co.batchsize))
    raise ValueError("Unknown mode! " + str(opt.mode))  # "options.mode not recognized!" (distri_client.h:294)
