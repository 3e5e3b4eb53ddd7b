"""The plane-digest test network (tests/planenet.py) pinned to its definition: the torch restatement of
oracles.fakenet bit for bit on 2^20 keys (its splitmix64 relies on wrapping int64 multiplication and
masked logical shifts), the same digest from every leaf-batch layout, and the checks that make a wrong
plane writer visible.  On CPU tensors here; the `gpu` parameters run the same on CUDA tensors."""
import numpy as np
import pytest
import torch

from tests import oracles, planenet

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]


def _keys():
    rng = np.random.default_rng(2026)
    edge = np.array([0, 1, 2, 0x5EED5EED, (1 << 31) - 1, 1 << 31, (1 << 32) - 1, 1 << 32, (1 << 63) - 1, 1 << 63,
                     (1 << 63) + 1, (1 << 64) - 2, (1 << 64) - 1], np.uint64)
    return np.concatenate([edge, rng.integers(0, 1 << 64, (1 << 20) - len(edge), dtype=np.uint64, endpoint=False)])


@pytest.mark.parametrize("device", DEVICES)
def test_torch_fakenet_equals_oracle_fakenet(device):
    """2^20 keys (0, 2^63, 2^64-1 and the other edges of the shifts and of the sign bit among them) through
    the 9x9 head, and 2^14 of them through the full 19x19 head: pi and V bit for bit"""
    keys = _keys()
    for A, chunk, count in ((82, 1 << 17, len(keys)), (362, 1 << 14, 1 << 14)):
        for lo in range(0, count, chunk):
            k = keys[lo: lo + chunk]
            pi, v = oracles.fakenet(k, A)
            tp, tv = planenet.fakenet_torch(torch.from_numpy(k.view(np.int64)).to(device), A)
            np.testing.assert_array_equal(tp.cpu().numpy().view(np.uint32), pi.view(np.uint32))
            np.testing.assert_array_equal(tv.cpu().numpy().view(np.uint32), v.view(np.uint32))


def _positions(n, count, seed):
    """float32 [count, 18, n, n]: AGZ planes of random games under all D4 codes (history planes filled)"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(count):
        o = oracles.Oracle(n)
        for _ in range(int(rng.integers(0, 3 * n * n // 2))):
            lg = np.flatnonzero(o.legal())
            if len(lg) == 0 or o.terminated():
                break
            o.forward(int(rng.choice(lg)))
        out.append(o.features(i % 8))
    return np.stack(out)


def _layouts(x, device):
    """the same planes as the three leaf-batch layouts of the search"""
    t = torch.from_numpy(x).to(device)
    nhwc = t.permute(0, 2, 3, 1)
    pad = lambda c, dt: torch.cat([nhwc, torch.zeros(*nhwc.shape[:3], c - 18, device=device)], 3).to(dt)  # noqa: E731
    return {"f32": {"s": t.contiguous()}, "f16": {"s_nhwc": pad(24, torch.float16).contiguous()},
            "bf16": {"s_nhwc": pad(32, torch.bfloat16).contiguous()}}


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("n", [9, 19])
def test_digest_is_the_same_in_every_layout(n, device):
    """float32 NCHW, f16 NHWC cpad 24 and bf16 NHWC cpad 32 give the numpy twin's digest and answer; the
    chunked sums give the unchunked ones; the numpy callback answers oracles.fakenet of the digest"""
    x = _positions(n, 40, n)
    x = np.concatenate([x, np.zeros((1, 18, n, n), np.float32), np.ones((1, 18, n, n), np.float32)])
    want = planenet.digest_np(x)
    assert len(set(want.tolist())) == len(x)  # 42 different positions, 42 digests
    pi, v = oracles.fakenet(want, n * n + 1)
    cp, cv = planenet.callback(x, None)
    np.testing.assert_array_equal(cp, pi)
    np.testing.assert_array_equal(cv, v)
    for chunk in (8192, 7):
        net = planenet.PlaneNet(n, device, chunk=chunk)
        for name, batch in _layouts(x, device).items():
            d = net.digest(batch).cpu().numpy().view(np.uint64)
            np.testing.assert_array_equal(d, want, err_msg=name)
            r = net(batch)
            np.testing.assert_array_equal(r["pi"].cpu().numpy(), pi, err_msg=name)
            np.testing.assert_array_equal(r["V"].cpu().numpy(), v, err_msg=name)
        assert int(net.bad) == 0 and net.calls == 3


@pytest.mark.parametrize("device", DEVICES)
def test_digest_sees_every_plane_value_and_the_padding(device):
    """one flipped entry in any plane, or a 1 in the NHWC padding, changes the digest; a value outside
    {0, 1} anywhere (padding included) is counted by the torch twin and refused by the numpy twin"""
    n = 9
    x = _positions(n, 4, 1)
    net = planenet.PlaneNet(n, device)
    base = planenet.digest_np(x)
    rng = np.random.default_rng(0)
    for _ in range(64):
        c, i, j = int(rng.integers(18)), int(rng.integers(n)), int(rng.integers(n))
        y = x.copy()
        y[1, c, i, j] = 1 - y[1, c, i, j]
        d = net.digest({"s": torch.from_numpy(y).to(device)}).cpu().numpy().view(np.uint64)
        assert d[1] != base[1] and (d[[0, 2, 3]] == base[[0, 2, 3]]).all(), (c, i, j)
    for fmt in ("f16", "bf16"):
        b = _layouts(x, device)[fmt]["s_nhwc"]
        b[2, 3, 4, 20] = 1
        d = net.digest({"s_nhwc": b}).cpu().numpy().view(np.uint64)
        assert d[2] != base[2] and (d[[0, 1, 3]] == base[[0, 1, 3]]).all()
        assert int(net.bad) == 0
        b[0, 0, 0, 23] = 0.5
        net.digest({"s_nhwc": b})
        assert int(net.bad) == 1
        net.bad.zero_()
    y = x.copy()
    y[0, 5, 0, 0] = 2
    with pytest.raises(AssertionError, match="outside"):
        planenet.digest_np(y)
