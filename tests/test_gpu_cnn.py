"""wgmma GEMM + ResNet-101-FPN backbone (csrc/mf_cnn.cu) against a plain PyTorch fp32 reference of the
same ops with the same (seeded, bf16-representable) weights.  The reference's real network lives in an
un-vendored third party (matterport Mask_RCNN + COCO weights + TF 1.8: "parity unpinned", SURVEY 8c), so
parity here = agreement with the PyTorch restatement of the published architecture.
Tolerance: activations are stored in bf16 between layers (8 mantissa bits => 2^-8 relative per rounding);
the reference applies the same bf16 rounding between layers, accumulation is fp32 on both sides."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _gemm(mfb, torch, M, N, K, relu, use_res, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    B = (torch.randn(N, K, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    R = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16) if use_res else None
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    L = mfb.load_library()
    rc = L.mf_gemm_bf16(C.c_void_p(A.data_ptr()), C.c_void_p(B.data_ptr()), C.c_void_p(bias.data_ptr()),
                        C.c_void_p(R.data_ptr()) if use_res else None, C.c_void_p(out.data_ptr()), M, N, K, int(relu),
                        C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, L.mf_cnn_last_error().decode()
    torch.cuda.synchronize()
    ref = A.float() @ B.float().t() + bias[None, :]
    if use_res:
        ref = ref + R.float()
    if relu:
        ref = torch.relu(ref)
    err = (out.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    return err, scale, bool(torch.isnan(out.float()).any())


@pytest.mark.parametrize("M,N,K,relu,res", [(128, 64, 64, 0, 0), (256, 128, 64, 0, 0), (1024, 64, 192, 1, 0), (4096, 256, 576, 1, 1),
                                            (65536, 64, 64, 1, 0), (1024, 2048, 512, 1, 1), (200, 128, 128, 0, 1),
                                            (32768, 256, 128, 1, 1)])                  # >= 132 tiles of 128 columns: BN = 128
def test_gemm_matches_torch(M, N, K, relu, res):
    import torch
    import maskfusion_b200 as mfb
    err, scale, has_nan = _gemm(mfb, torch, M, N, K, relu, res, seed=M + N + K)
    assert not has_nan
    assert err <= 2.0 ** -7 * max(scale, 1.0), (err, scale)       # one bf16 rounding of the output (fp32 accumulate on both sides)


@pytest.mark.parametrize("H,W,Cin,Cout", [(256, 256, 64, 64), (128, 128, 128, 128), (64, 64, 256, 256), (32, 32, 512, 512), (16, 16, 256, 256),
                                         (256, 256, 64, 128)])                         # 512 M tiles x 1: BN = 128
def test_implicit_conv3x3_matches_torch(H, W, Cin, Cout):
    """3x3/s1/p1 convolution through the 3-D TMA map (zero fill == padding), tiles of 128 / (64x2) / (32x4) / (16x8) pixels"""
    import torch
    import torch.nn.functional as F
    import maskfusion_b200 as mfb
    g = torch.Generator(device="cuda").manual_seed(H + Cin)
    x = torch.randn(H, W, Cin, device="cuda", generator=g).to(torch.bfloat16).contiguous()
    w = (torch.randn(Cout, 3, 3, Cin, device="cuda", generator=g) * (2.0 / (9 * Cin)) ** 0.5).to(torch.bfloat16).contiguous()
    bias = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(H, W, Cout, device="cuda", generator=g).to(torch.bfloat16).contiguous()
    out = torch.full((H, W, Cout), float("nan"), device="cuda", dtype=torch.bfloat16)
    L = mfb.load_library()
    rc = L.mf_conv3x3_bf16(C.c_void_p(x.data_ptr()), C.c_void_p(w.data_ptr()), C.c_void_p(bias.data_ptr()), C.c_void_p(res.data_ptr()),
                           C.c_void_p(out.data_ptr()), H, W, Cin, Cout, 1, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, L.mf_cnn_last_error().decode()
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(2, 0, 1)[None], w.float().permute(0, 3, 1, 2), bias, padding=1)[0].permute(1, 2, 0) + res.float()
    ref = torch.relu(ref)
    assert not torch.isnan(out.float()).any()
    assert (out.float() - ref).abs().max().item() <= 2.0 ** -7 * max(ref.abs().max().item(), 1.0)


def _torch_backbone(torch, bb, x_nhwc_bf16):
    """PyTorch restatement of resnet_graph(resnet101, stage5) + FPN (matterport mrcnn/model.py) with bf16 storage between layers"""
    import torch.nn.functional as F
    layers = bb.layers()

    def conv(i, x, residual=None, relu=True):
        cin, cout, k, stride, pad, kpad = layers[i]
        w, b = bb.weights(i)
        wt = torch.from_numpy(w).cuda().permute(0, 3, 1, 2).contiguous()          # [cout, cin, kh, kw]
        y = F.conv2d(x.float(), wt, torch.from_numpy(b).cuda(), stride=stride, padding=pad)
        if residual is not None:
            y = y + residual.float()
        if relu:
            y = torch.relu(y)
        return y.to(torch.bfloat16)

    x = x_nhwc_bf16.permute(2, 0, 1)[None]                                         # NCHW
    li = 0
    x = conv(li, x); li += 1
    x = F.max_pool2d(F.pad(x.float(), (0, 1, 0, 1), value=float("-inf")), 3, 2).to(torch.bfloat16)
    Cs = []
    for st, nb in enumerate((3, 4, 23, 3)):
        for blk in range(nb):
            a = conv(li, x); b = conv(li + 1, a)
            if blk == 0:
                sc = conv(li + 3, x, relu=False); nl = li + 4
            else:
                sc = x; nl = li + 3
            x = conv(li + 2, b, residual=sc, relu=True)
            li = nl
        Cs.append(x)
    lat = [li + i for i in range(4)]; outc = [li + 4 + i for i in range(4)]
    top = conv(lat[3], Cs[3], relu=False)
    P = [None] * 5
    P[3] = conv(outc[3], top, relu=False)
    for i in (2, 1, 0):
        l = conv(lat[i], Cs[i], relu=False)
        top = (l.float() + F.interpolate(top.float(), scale_factor=2, mode="nearest")).to(torch.bfloat16)
        P[i] = conv(outc[i], top, relu=False)
    P[4] = P[3][:, :, ::2, ::2]
    return Cs, P


def test_backbone_matches_torch():
    import torch
    import maskfusion_b200 as mfb
    S = 256
    bb = mfb.Backbone(S, seed=7, stream=torch.cuda.current_stream().cuda_stream)
    assert len(bb.layers()) == 1 + 33 * 3 + 4 + 8
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.randn(S, S, 3, device="cuda", generator=g) * 60.0).to(torch.bfloat16).contiguous()
    bb.forward(x.data_ptr())
    torch.cuda.synchronize()
    Cs, P = _torch_backbone(torch, bb, x)
    report = {}
    for lvl in range(9):
        got = torch.from_numpy(bb.download(lvl)).cuda()
        ref = (Cs[lvl] if lvl < 4 else P[lvl - 4])[0].permute(1, 2, 0).float()
        assert not torch.isnan(got).any(), lvl
        denom = ref.abs().mean().item() + 1e-6
        report[lvl] = ((got - ref).abs().mean().item() / denom, ref.abs().mean().item())
    # bf16 storage: errors random-walk over ~100 layers; mean relative error stays at the percent level
    for lvl, (rel, mag) in report.items():
        assert mag > 1e-3, (lvl, "degenerate activations", report)
        assert rel < 0.06, report
    assert bb.numGemms() == 112
    bb.close()
