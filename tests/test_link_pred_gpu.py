"""GPU tests of the end-of-epoch quality line (csrc/eval.cu) against numpy statements, exactly:
  - gg_pair_dot_f64 is the float64 dot in the kernel's order (per lane g: sequential adds over the float4 chunks
    g, g + 8, ...; then the xor-4, 2, 1 butterfly), and within gamma_n sum|products| of the exact dot;
  - gg_link_pred_acc gives np.median and the accuracy of (score >= median) against [1] * (n // 2) + [0] * (n - n // 2),
    at the sizes and values where a radix select goes wrong: ties, -0 / +0, infinities, subnormals, keys that share
    their top seven bytes, the middle pair across the sign boundary, and NaN."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _dot_order(A, B):
    """gg_pair_dot_f64's sums in numpy (A, B: float32 [P, ld])."""
    ld = A.shape[1]
    a = A.astype(np.float64).reshape(len(A), ld // 32, 8, 4)
    b = B.astype(np.float64).reshape(len(B), ld // 32, 8, 4)
    s = np.zeros((len(A), 8))
    for c in range(ld // 32):
        for k in range(4):
            s = s + a[:, c, :, k] * b[:, c, :, k]          # the fp64 product of two fp32 values is exact
    for off in (4, 2, 1):
        s = s + s[:, np.arange(8) ^ off]
    return s[:, 0]


@pytest.mark.parametrize("ld", [32, 64, 128, 256, 512])
def test_pair_dot_f64_is_the_kernel_order(ld, cuda_device):
    import torch
    from graphgan_b200 import _cabi
    rs = np.random.RandomState(ld)
    n, P = 500, 4099
    E = np.zeros((n, ld), np.float32)
    E[:, :ld - 5] = rs.normal(0, 1, size=(n, ld - 5)) * 10.0 ** rs.randint(-6, 7, size=(n, 1))
    E[:40, :ld - 5] = np.abs(E[:40, :ld - 5]) * np.where(np.arange(ld - 5) % 2, -1, 1)    # heavy cancellation
    i, j = rs.randint(0, n, P).astype(np.int32), rs.randint(0, n, P).astype(np.int32)
    i[:100], j[:100] = rs.randint(0, 40, 100), rs.randint(0, 40, 100)
    to = lambda x: torch.as_tensor(x).to(cuda_device)
    out = torch.empty(P, dtype=torch.float64, device=cuda_device)
    emb, di, dj = to(E), to(i), to(j)
    _cabi.check(_cabi.lib().gg_pair_dot_f64(P, di.data_ptr(), dj.data_ptr(), emb.data_ptr(), ld, out.data_ptr(), None),
                "gg_pair_dot_f64")
    got = out.cpu().numpy()
    want = _dot_order(E[i], E[j])
    assert np.array_equal(got.view(np.int64), want.view(np.int64))
    prod = E[i].astype(np.float64) * E[j].astype(np.float64)
    exact = np.array([math.fsum(r) for r in prod])
    k = ld // 8 + 3
    gam = k * 2.0 ** -53 / (1 - k * 2.0 ** -53)
    assert np.all(np.abs(got - exact) <= gam * np.abs(prod).sum(1))


def _ref(score):
    """The reference's quality line (link_prediction.py:27-36): median, then accuracy_score of (score >= median)."""
    med = np.median(score)
    n = len(score)
    truth = np.zeros(n)
    truth[:n // 2] = 1
    return float(np.mean((score >= med).astype(np.float64) == truth)), float(med)


def _device(score, dev):
    import torch
    from graphgan_b200 import _cabi
    s = torch.as_tensor(np.ascontiguousarray(score, np.float64)).to(dev)
    out = torch.full((2,), 7.0, dtype=torch.float64, device=dev)
    _cabi.check(_cabi.lib().gg_link_pred_acc(len(score), s.data_ptr(), out.data_ptr(), None), "gg_link_pred_acc")
    acc, med = out.cpu().numpy()
    return float(acc), float(med)


def _cases():
    rs = np.random.RandomState(11)
    out = {}
    for n in (1, 2, 3, 1023, 1024, 1025, 2 ** 20 + 1):
        out["random_%d" % n] = rs.normal(0, 1, n)
    out["all_equal"] = np.full(1000, 0.375)
    t = rs.normal(0, 1, 2001)
    t[500:1700] = 0.25                                      # heavy ties across the median
    out["ties"] = t
    out["ties_even"] = np.concatenate([t, [0.25]])
    z = rs.normal(0, 1, 1000)
    z[::3] = 0.0
    z[1::3] = -0.0
    out["signed_zeros"] = z
    out["zero_pair"] = np.array([-0.0, 0.0])
    out["zero_pair_rev"] = np.array([0.0, -0.0, -0.0])
    inf = rs.normal(0, 1, 999)
    inf[:300] = np.inf
    inf[300:500] = -np.inf
    out["infinities"] = inf
    out["inf_middle"] = np.array([np.inf, -np.inf, 1.0, -1.0, np.inf, -np.inf])          # median of -1 and 1
    out["inf_straddle"] = np.array([np.inf, -np.inf])                                    # mean of -inf and inf: NaN
    tiny = np.finfo(np.float64).tiny
    sub = rs.randint(1, 1000, 1001) * 5e-324 * rs.choice([-1, 1], 1001)
    sub[:5] = [5e-324, -5e-324, tiny, -tiny, 0.0]
    out["subnormals"] = sub
    base = np.float64(1.5).view(np.int64)
    out["top7_shared"] = (base + rs.randint(0, 256, 4097)).view(np.float64)                 # only the last byte differs
    neg = np.float64(-2.75).view(np.int64)
    out["top7_shared_neg"] = (neg + rs.randint(0, 256, 2048)).view(np.float64)
    out["sign_boundary"] = np.concatenate([-rs.random_sample(500) - 1e-300, rs.random_sample(500) + 1e-300])
    out["sign_boundary_tiny"] = np.concatenate([np.full(500, -5e-324), np.full(500, 5e-324)])
    return out


@pytest.mark.parametrize("name", sorted(_cases()))
def test_link_pred_acc_equals_numpy(name, cuda_device):
    score = _cases()[name]
    want = _ref(score)
    got = _device(score, cuda_device)
    assert got[0] == want[0], (got, want)
    assert got[1] == want[1] or (math.isnan(got[1]) and math.isnan(want[1])), (got, want)


@pytest.mark.parametrize("n,where", [(1, [0]), (2, [1]), (1025, [3]), (1024, [0, 1000]), (4097, [2048])])
def test_link_pred_acc_with_nan_matches_the_reference(n, where, cuda_device):
    """A diverged model's NaN score makes np.median NaN, every (score >= median) False and the accuracy (n - n // 2) / n.
    The device must write that line, not a median over the other scores."""
    rs = np.random.RandomState(n)
    score = rs.normal(0, 1, n)
    score[where] = np.nan
    if len(where) > 1:
        score[where[1]] = -np.nan
    want = _ref(score)
    assert math.isnan(want[1]) and want[0] == (n - n // 2) / n
    got = _device(score, cuda_device)
    assert got[0] == want[0] and math.isnan(got[1]), got
