"""Proposal generation on a canvas whose P2 level holds more anchors than 64 selection chunks of 4096 (1408x2048: 540 672 on P2),
teacher-forced with seeded RPN maps and compared level by level with the oracle's generate_proposals_level."""
import numpy as np
import pytest
import torch

H, W, B = 1408, 2048, 2
PRE, POST, NMS = 1000, 1000, 0.7


def _rpn_maps(h, w, A, seed, quantised):
    """Objectness [A,h,w] and deltas [4A,h,w] (fp32).  The top PRE scores are distinct and cluster around a few centres so that the NMS
    has work.  continuous: every score is distinct, so the two-level radix select narrows the level to ~PRE keys.  quantised: every other
    anchor scores exactly 0.75 and the top PRE lie 1..PRE ulps above it, all in the same 22-bit key sub-bin: the boundary sub-bin then
    holds the whole level (> 8192 keys) and the level is sorted whole, while the top PRE still have no equal-score ties."""
    rng = np.random.RandomState(seed)
    n = A * h * w
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    bump = np.zeros((h, w))
    for cy, cx in zip(rng.uniform(0, h, 6), rng.uniform(0, w, 6)):
        bump += np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * (0.02 * h) ** 2))
    key = np.broadcast_to(bump, (A, h, w)).reshape(-1) + 1e-3 * rng.rand(n)
    rank = np.empty(n, np.int64)
    rank[np.argsort(-key, kind="stable")] = np.arange(n)          # 0 = best
    if quantised:
        s = np.full(n, 0.75, np.float32)
        top = rank < PRE
        s[top] = (0.75 + (PRE - rank[top]) * 2.0 ** -24).astype(np.float32)
    else:
        s = ((n - rank) / (n + 1.0)).astype(np.float32)
    assert len(np.unique(s[rank < PRE])) == PRE
    deltas = (0.3 * rng.randn(4 * A, h, w)).astype(np.float32)
    return torch.from_numpy(s.reshape(A, h, w)), torch.from_numpy(deltas)


@pytest.mark.gpu
@pytest.mark.parametrize("quantised", [False, True], ids=["continuous", "quantised"])
def test_fpn_proposals_large_levels(built, quantised):
    from detectorch_b200 import engine as E
    from oracle import network as net
    from oracle import ref
    dev = torch.device("cuda:0")
    eng = E.Engine(arch="resnet50", batch=B, height=H, width=W, pre_nms_top_n=PRE, post_nms_top_n=POST, rpn_nms_thresh=NMS, use_mask=False)
    eng.load_state_dict(net.synthetic_params("resnet50", mask=False))
    A = 3
    assert eng.buffer("rpn_out2").shape[1] * eng.buffer("rpn_out2").shape[2] * A > 64 * 4096
    maps = {}
    for b in range(B):
        for i in range(5):
            o = eng.buffer("rpn_out%d" % (i + 2))
            s, d = _rpn_maps(o.shape[1], o.shape[2], A, seed=10 * b + i, quantised=quantised)
            o[b, ..., 0:A] = s.permute(1, 2, 0).to(dev)
            o[b, ..., A:5 * A] = d.permute(1, 2, 0).to(dev)
            maps[b, i] = (s, d)
    eng.run(None, 1.0, E.ST_PROPOSALS, E.ST_COLLECT)
    torch.cuda.synchronize()
    for b in range(B):
        cnt = eng.buffer("prop_counts")[b].cpu().numpy()
        for i in range(5):
            s, d = maps[b, i]
            props, scores, st = ref.generate_proposals_level(s[None], d[None], H, W, 1.0, 1.0 / (4 << i), (32 << i,), pre_nms_top_n=PRE,
                                                             post_nms_top_n=POST, nms_thresh=NMS, return_stages=True)
            order = st["order"]
            assert np.array_equal(eng.buffer("rpn_order")[b, i, :len(order)].cpu().numpy(), order), (b, i)
            k = int(cnt[i])
            assert k == len(props), (b, i, k, len(props))
            assert torch.equal(eng.buffer("prop_scores")[b, i, :k].cpu(), scores[:, 0]), (b, i)
            assert (eng.buffer("props")[b, i, :k].cpu() - props).abs().max().item() <= 2e-4, (b, i)      # expf ulp
        assert int(eng.buffer("roi_counts")[b]) == min(POST, int(cnt.sum()))
