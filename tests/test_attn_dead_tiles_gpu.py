"""GPU (-m gpu): attention with a per-key bias whose 128-key tiles are -inf throughout ("dead" tiles) against the same
attention with those tiles removed from K, V and the bias.  The kernels skip dead tiles (ops.key_bias_live_list); a dead
tile adds p = 0 to every row, so skipping it must give the same bits as processing it: O, LSE and dQ equal bit for bit,
dK and dV equal on the live keys and exactly zero on the dead ones.  Every sample is compared with a run of its own
(its dead set differs), so the batched run is checked against B = 1 runs too."""
import pytest
import torch

from simpletuner_b200 import ops

pytestmark = pytest.mark.gpu
NEG = float("-inf")


def _bias(Sk, dead, extra_neg=(), seed=0):
    """[Sk] bias: finite values, -inf over the 128-key tiles in `dead` and at the key indices in `extra_neg`."""
    g = torch.Generator().manual_seed(seed)
    b = torch.randn(Sk, generator=g)
    for t in dead:
        b[128 * t:min(128 * (t + 1), Sk)] = NEG
    for i in extra_neg:
        b[i] = NEG
    return b.bfloat16()


def _keep(Sk, bias_row):
    """Key indices of the tiles that are not -inf throughout (the tiles the kernels keep)."""
    idx = []
    for t in range((Sk + 127) // 128):
        sl = slice(128 * t, min(128 * (t + 1), Sk))
        if not bool(torch.isneginf(bias_row[sl]).all()):
            idx += list(range(sl.start, sl.stop))
    return torch.tensor(idx)


def _run(q, k, v, d_o, bias):
    o, lse = ops.attn_fwd(q, k, v, key_bias=bias)
    dq, dk, dv = ops.attn_bwd(q, k, v, o, d_o, lse, key_bias=bias)
    torch.cuda.synchronize()
    return o, lse, dq, dk, dv


CASES = {
    # name: (HD, Sq, Sk, per-sample dead tile sets, per-sample extra -inf keys)
    "leading": (128, 640, 640, [(0, 1)], [()]),
    "trailing": (64, 512, 700, [(4, 5)], [()]),                       # the tail tile (60 keys) is dead
    "interleaved_b3": (128, 700, 1100, [(1, 3, 5), (0, 8), (2, 4, 6, 7)], [(), (1030,), ()]),
    "tail_live_partly_masked": (64, 300, 900, [(0, 2), (6,), (3,)], [tuple(range(770, 890)), (), tuple(range(768, 899))]),
    "chroma_like_b2": (128, 1536, 1536, [(1, 2, 3), (3,)], [tuple(range(100, 128)), tuple(range(300, 384))]),
}


@pytest.mark.parametrize("case", list(CASES))
def test_dead_tiles_give_the_bits_of_removing_them(case):
    HD, Sq, Sk, dead, extra = CASES[case]
    B, H = len(dead), 3
    g = torch.Generator().manual_seed(1)
    q, k, v, d_o = ((torch.randn(B, n, H, HD, generator=g) * 0.5).bfloat16().cuda() for n in (Sq, Sk, Sk, Sq))
    bias = torch.stack([_bias(Sk, dead[i], extra[i], seed=i) for i in range(B)]).cuda()
    full = _run(q, k, v, d_o, bias)
    for i in range(B):
        keep = _keep(Sk, bias[i].cpu()).cuda()
        sub = _run(q[i:i + 1], k[i:i + 1, keep].contiguous(), v[i:i + 1, keep].contiguous(), d_o[i:i + 1],
                   bias[i:i + 1, keep].contiguous())
        o, lse, dq, dk, dv = (t[i:i + 1] for t in full)
        assert torch.equal(o, sub[0]) and torch.equal(lse, sub[1]) and torch.equal(dq, sub[2]), (case, i)
        assert torch.equal(dk[:, keep], sub[3]) and torch.equal(dv[:, keep], sub[4]), (case, i)
        dead_keys = torch.ones(Sk, dtype=torch.bool, device="cuda")
        dead_keys[keep] = False
        assert not dk[:, dead_keys].any() and not dv[:, dead_keys].any(), (case, i)


@pytest.mark.parametrize("HD", [64, 128])
def test_shared_bias_row(HD):
    B, H, S = 2, 2, 900
    g = torch.Generator().manual_seed(2)
    q, k, v, d_o = ((torch.randn(B, S, H, HD, generator=g) * 0.5).bfloat16().cuda() for _ in range(4))
    bias = _bias(S, (1, 4, 7), seed=5)[None].cuda()           # [1, Sk]: one row for the batch
    full = _run(q, k, v, d_o, bias)
    keep = _keep(S, bias[0].cpu()).cuda()
    sub = _run(q, k[:, keep].contiguous(), v[:, keep].contiguous(), d_o, bias[:, keep].contiguous())
    assert all(torch.equal(a, b) for a, b in zip(full[:3], sub[:3]))
    assert torch.equal(full[3][:, keep], sub[3]) and torch.equal(full[4][:, keep], sub[4])
    assert int(ops.key_bias_live_list(bias)[0, 0]) == 5


def test_live_list_is_built_once_per_bias():
    bias = _bias(600, (0, 2)).cuda()[None]
    l1 = ops._key_live(bias)
    assert ops._key_live(bias) is l1
    assert l1.tolist() == [[3, 1, 3, 4, 0, 2, 0, 1, 0, 1, 1]]
