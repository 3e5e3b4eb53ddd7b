"""A deterministic test network that reads the leaf PLANES (test infrastructure only).

``oracles.fakenet`` is keyed by a 64-bit number; the search tests usually key it by the leaf's position
hash, fetched on the host for every leaf.  That skips the leaf planes, and at full size (32,768 leaves
of 361 points per wave) it costs a host round trip per wave.  This net keys ``oracles.fakenet`` by an
exact integer digest of the planes instead, as a pure function of what the search hands a network: a
wrong plane changes the priors, and the root visit tables show it.

Digest: the "value == 1" indicator of every plane entry, dotted with fixed 31-bit weights, as two
independent int64 sums ``s1``, ``s2`` (each < 2^31 * 32 * 361 < 2^45, so no overflow) folded into 64 bits
as ``(s1 << 32) ^ s2``.  Integer sums do not depend on the order of summation, so the digest is
bit-equal on any device.  Weights exist for 32 channels: the digest covers the zero padding of the
channels-last formats too (channels >= 18), which the host twin, holding only the 18 planes, counts as
zero -- a writer that leaves non-zero padding therefore changes the digest.  Values outside {0, 1} are
counted (``PlaneNet.bad``, a device scalar read once at the end of a run).

Two twins:
* ``PlaneNet``: torch, on the tensors' device and the caller's stream, no host synchronisation; the
  network callback of ``MctsBatch`` / ``WavePipeline`` (``batch["s"]`` float32 NCHW or ``batch["s_nhwc"]``
  float16 / bfloat16 NHWC with 24 or 32 channels).
* ``callback``: numpy, the ``callback(feats, hashes)`` of ``oracles.OracleMcts`` / ``oracles.RefMcts``.
Both answer ``oracles.fakenet(digest, N*N+1)``; the torch restatement of it is pinned bit for bit by
``tests/test_planenet.py``."""
import numpy as np
import torch

from tests import oracles

CMAX = 32  # channels the weights cover (the widest padded layout)
_M64 = 1 << 64


def weights(n):
    """int64 [2, CMAX, n, n]: the 31-bit weights of the two digest sums, by (channel, row, column)"""
    i = np.arange(2 * CMAX * n * n, dtype=np.uint64) + np.uint64(n << 32)
    return (oracles._splitmix64(i) >> np.uint64(33)).astype(np.int64).reshape(2, CMAX, n, n)


def digest_np(planes):
    """uint64 [m]: the digest of float planes [m, C, n, n] (C <= CMAX), channel-first"""
    x = np.asarray(planes)
    m, C, n, _ = x.shape
    bad = ~((x == 0) | (x == 1))
    if bad.any():
        raise AssertionError(f"{int(bad.sum())} plane values outside {{0, 1}}")
    ind = (x == 1).reshape(m, -1).astype(np.int64)
    W = weights(n)[:, :C].reshape(2, -1)
    s1, s2 = (ind @ W[0]).astype(np.uint64), (ind @ W[1]).astype(np.uint64)
    return (s1 << np.uint64(32)) ^ s2


def callback(feats, hashes=None):
    """``callback(feats [m,18,n,n] float32, hashes)`` for OracleMcts / RefMcts: (pi [m,N*N+1], v [m])"""
    n = feats.shape[-1]
    return oracles.fakenet(digest_np(feats), n * n + 1)


# -- torch restatement of oracles.fakenet on int64 tensors (two's complement wrap-around) --------------
def _s64(c):
    """the int64 with the bit pattern of the uint64 constant c"""
    return c - _M64 if c >= 1 << 63 else c


_GOLD = _s64(0x9E3779B97F4A7C15)
_MUL1 = _s64(0xBF58476D1CE4E5B9)
_MUL2 = _s64(0x94D049BB133111EB)


def _srl(x, k):
    """logical right shift of an int64 tensor (>> is arithmetic on signed tensors)"""
    return (x >> k) & ((1 << (64 - k)) - 1)


def _splitmix64(x):
    x = x + _GOLD
    x = (x ^ _srl(x, 30)) * _MUL1
    x = (x ^ _srl(x, 27)) * _MUL2
    return x ^ _srl(x, 31)


def fakenet_torch(keys, num_actions):
    """keys: int64 tensor [m] (the uint64 bit patterns) -> (pi float32 [m, A], v float32 [m]), bit-equal
    to oracles.fakenet"""
    a = torch.arange(1, num_actions + 1, dtype=torch.int64, device=keys.device) * _GOLD
    r = _splitmix64(keys[:, None] ^ a[None, :])
    u = (_srl(r, 40) + 1).to(torch.float32) * (1.0 / 16777216.0)
    t = u * u
    t = t * t
    t = t * t
    r2 = _splitmix64(keys ^ 0x5EED5EED)
    v = _srl(r2, 40).to(torch.float32) * (1.0 / 8388608.0) - 1.0
    return t, v


class PlaneNet:
    """``net(batch) -> {"pi", "V"}`` computed from the planes on their device.  ``batchsize``: the
    search pads its leaf batch to a multiple of it (``MctsBatch.wave_select``), as the bench's
    ``FusedActor`` asks; 0 = no padding."""

    def __init__(self, n, device, batchsize=256, chunk=8192):
        self.n, self.batchsize, self.chunk = n, batchsize, chunk
        self.W = torch.from_numpy(weights(n)).to(device)
        self.bad = torch.zeros((), dtype=torch.int64, device=device)  # values outside {0, 1}, all calls
        self.calls = 0

    def digest(self, batch):
        """int64 [m] digests of ``batch["s"]`` (float32 [m,C,n,n]) or ``batch["s_nhwc"]`` ([m,n,n,C])"""
        if "s" in batch:
            x = batch["s"]
            W = self.W[:, : x.shape[1]]
        else:
            x = batch["s_nhwc"]
            W = self.W[:, : x.shape[3]].permute(0, 2, 3, 1)
        assert x.shape[1:] == W.shape[1:], (tuple(x.shape), tuple(W.shape))
        out = torch.empty(x.shape[0], dtype=torch.int64, device=x.device)
        zero = torch.zeros((), dtype=torch.int64, device=x.device)
        for lo in range(0, x.shape[0], self.chunk):  # bounds the int64 temporaries
            xc = x[lo: lo + self.chunk]
            one = xc == 1
            self.bad += ((xc != 0) & ~one).sum()
            s1 = torch.where(one, W[0], zero).flatten(1).sum(1)
            s2 = torch.where(one, W[1], zero).flatten(1).sum(1)
            out[lo: lo + self.chunk] = (s1 << 32) ^ s2
        return out

    def __call__(self, batch):
        self.calls += 1
        pi, v = fakenet_torch(self.digest(batch), self.n * self.n + 1)
        return {"pi": pi, "V": v}
