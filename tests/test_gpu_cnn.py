"""wgmma GEMM, implicit 3x3 convolution and input mould (csrc/mf_cnn.cu), and the ResNet-101-FPN backbone.

GEMM and convolution are pinned bit for bit on integer operands: every product and every partial sum is an integer of magnitude at most
2^20, so fp32 accumulation is exact in any order, bias and residual are integers too, and the only rounding left is the epilogue's bf16
round-to-nearest-even, compared as a bit pattern with the exact float64 result rounded to bf16.  Two operand classes:
  dense  entries in [-8, 8]: |product| <= 64, so K up to 12 544 (FC1) stays below 2^20;
  full   A in [-255, 255] (every bf16 mantissa bit of an integer), each B row at most 16 nonzeros in [-255, 255], placed in the first and last
         k-block and the blocks around the 4-stage ring's wrap (3, 4, 5, 8): a k-block mapped, waited on or released wrongly, or dropped low
         mantissa bits, change the result.
The shapes sweep the tile logic (M tails, BN = 64 / 128 at the SM-count boundary, N, K / 64 through the ring wrap, relu with negative sums,
residual on and off; conv boxes Wbox 8..128 x Hbox 16..1, 1..3 boxes per row, cblocks 1..8).  Every output gets 128 extra rows of NaN that
must stay untouched.

The mould is pinned bit for bit against R-MOLD (tests/heads_ref.mold_input).  The backbone is compared with a PyTorch restatement of the
published architecture on seeded weights (the reference's network is an un-vendored third party, SURVEY 8c) within a bf16 tolerance:
activations are stored in bf16 between layers on both sides, accumulation is fp32 on both sides."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from tests import heads_ref as ref

pytestmark = pytest.mark.gpu

CANARY = 128
RING_BLOCKS = (0, 3, 4, 5, 8)          # the first k-block and those around the first wraps of the 4-slot ring; the last is added per K


def _sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ints(torch, g, shape, lo, hi, nonzero=False):
    """uniform integers in [lo, hi] (nonzero: |v| in [1, hi], random sign) as float32"""
    if not nonzero:
        return torch.randint(lo, hi + 1, shape, device="cuda", generator=g).float()
    mag = torch.randint(1, hi + 1, shape, device="cuda", generator=g).float()
    return torch.where(torch.rand(shape, device="cuda", generator=g) < 0.5, -mag, mag)


def _sparse_rows(torch, g, N, K):
    """the full class's B: N x K, at most 16 nonzeros in [-255, 255] per row, spread round-robin over RING_BLOCKS and the last k-block"""
    nk = K // 64
    blocks = sorted({b for b in RING_BLOCKS if b < nk} | {nk - 1})
    blk = torch.tensor([blocks[j % len(blocks)] for j in range(16)], device="cuda")
    cols = blk[None, :] * 64 + torch.randint(0, 64, (N, 16), device="cuda", generator=g)
    B = torch.zeros(N, K, device="cuda")
    B.scatter_(1, cols, _ints(torch, g, (N, 16), -255, 255, nonzero=True))
    return B


def _operands(torch, g, cls, rowsA, N, K):
    if cls == "dense":
        return _ints(torch, g, (rowsA, K), -8, 8), _ints(torch, g, (N, K), -8, 8)
    return _ints(torch, g, (rowsA, K), -255, 255), _sparse_rows(torch, g, N, K)


def _epilogue_operands(torch, g, M, N, res):
    bias = _ints(torch, g, (N,), -1024, 1024)
    R = _ints(torch, g, (M, N), -256, 256).to(torch.bfloat16) if res else None
    return bias, R


def _canvas(torch, M, N):
    return torch.full((M + CANARY, N), float("nan"), device="cuda", dtype=torch.bfloat16)


def _check_exact(torch, out, exact, M, relu):
    """out [M + CANARY, N] bf16 against the exact float64 result [M, N]: bit patterns (+0 and -0 count as equal), canary rows untouched"""
    assert exact.abs().max().item() <= 2 ** 20
    if relu:
        assert (exact < 0).any(), "relu needs negative sums to show"
        exact = exact.clamp_min(0)
    want = exact.to(torch.bfloat16).view(torch.int16)
    got = out[:M].view(torch.int16)
    same = (got == want) | (((got & 0x7FFF) == 0) & ((want & 0x7FFF) == 0))
    bad = (~same).nonzero()
    assert bad.numel() == 0, (f"{bad.shape[0]} of {same.numel()} differ; first (row, col): {bad[:4].tolist()}; got "
                              f"{out[:M][tuple(bad[:4].t())].tolist()}, exact {exact[tuple(bad[:4].t())].tolist()}")
    nan = torch.full((1,), float("nan"), dtype=torch.bfloat16, device="cuda").view(torch.int16)
    assert (out[M:].view(torch.int16) == nan).all(), "rows >= M were written"


def _lib_call(torch, fn, *args):
    import maskfusion_b200 as mfb
    L = mfb.load_library()
    ptrs = [C.c_void_p(a.data_ptr()) if a is not None else None for a in args[:5]]
    rc = getattr(L, fn)(*ptrs, *args[5:], C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, L.mf_cnn_last_error().decode()
    torch.cuda.synchronize()


# (M, N, K, relu, residual, class); M as "sms-1" / "sms-1+1" is 128 (SMs - 1) and one row more with N = 128: the last M-tile count that
# takes BN = 64 and the first that takes BN = 128 on the card that runs the test
GEMM_CASES = [
    (1, 64, 64, 0, 0, "dense"), (64, 128, 128, 1, 1, "full"), (127, 192, 320, 0, 1, "dense"), (128, 64, 64, 0, 0, "dense"),
    (129, 448, 576, 1, 0, "full"), (200, 128, 128, 0, 1, "dense"), (256, 128, 64, 0, 0, "full"), (512, 1024, 256, 0, 1, "full"),
    (1000, 1024, 12544, 1, 0, "dense"), (1000, 448, 12544, 0, 1, "full"), (1024, 64, 192, 1, 0, "dense"), (1024, 2048, 512, 1, 1, "dense"),
    (1000, 2048, 320, 0, 0, "full"), (4096, 256, 576, 1, 1, "full"), (19600, 256, 2304, 1, 0, "full"), (19600, 1024, 256, 0, 1, "dense"),
    (32768, 256, 128, 1, 1, "full"), (65536, 64, 64, 1, 0, "dense"), (65536, 128, 320, 0, 1, "full"),
    ("sms-1", 128, 320, 1, 1, "dense"), ("sms-1+1", 128, 320, 1, 1, "dense"), ("sms-1", 128, 576, 0, 0, "full"), ("sms-1+1", 128, 576, 0, 0, "full"),
]


@pytest.mark.parametrize("M,N,K,relu,res,cls", GEMM_CASES)
def test_gemm_exact(M, N, K, relu, res, cls):
    import torch
    if isinstance(M, str):
        M = 128 * (_sms(torch) - 1) + (1 if M.endswith("+1") else 0)
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    A, B = _operands(torch, g, cls, M, N, K)
    bias, R = _epilogue_operands(torch, g, M, N, res)
    out = _canvas(torch, M, N)
    _lib_call(torch, "mf_gemm_bf16", A.to(torch.bfloat16), B.to(torch.bfloat16), bias, R, out, M, N, K, int(relu))
    exact = A.double() @ B.double().t() + bias.double()[None, :]
    if res:
        exact = exact + R.double()
    _check_exact(torch, out, exact, M, relu)


# (H, W, Cin, Cout, relu, residual, class): Wbox x Hbox = 8x16, 16x8, 32x4, 64x2, 128x1 and 2 or 3 boxes per row at W = 256, 384
CONV_CASES = [
    (16, 8, 64, 64, 1, 1, "dense"), (64, 16, 192, 128, 0, 0, "full"), (48, 32, 512, 192, 1, 0, "dense"), (96, 64, 64, 256, 0, 1, "full"),
    (128, 128, 192, 64, 1, 1, "dense"), (8, 256, 512, 128, 0, 1, "full"), (2, 384, 192, 256, 1, 0, "dense"), (256, 256, 64, 128, 1, 1, "full"),
    (256, 256, 64, 64, 1, 1, "dense"), (128, 128, 128, 128, 1, 1, "full"), (64, 64, 256, 256, 1, 1, "dense"), (32, 32, 512, 512, 1, 1, "full"),
    (16, 16, 256, 256, 1, 1, "dense"),
]


@pytest.mark.parametrize("H,W,Cin,Cout,relu,res,cls", CONV_CASES)
def test_implicit_conv3x3_exact(H, W, Cin, Cout, relu, res, cls):
    """3x3/s1/p1 convolution through the 3-D TMA map (its zero fill is the padding) against F.unfold + matmul in float64; no input pixel
    is 0, so a wrong tap or padding shows"""
    import torch
    import torch.nn.functional as F
    M, K = H * W, 9 * Cin
    g = torch.Generator(device="cuda").manual_seed(H * 31 + W * 7 + Cin + Cout)
    hi = 8 if cls == "dense" else 255
    x = _ints(torch, g, (H, W, Cin), -hi, hi, nonzero=True)
    w = _ints(torch, g, (Cout, K), -8, 8) if cls == "dense" else _sparse_rows(torch, g, Cout, K)     # K order (ky, kx, cin)
    bias, R = _epilogue_operands(torch, g, M, Cout, res)
    out = _canvas(torch, M, Cout)
    _lib_call(torch, "mf_conv3x3_bf16", x.to(torch.bfloat16), w.to(torch.bfloat16), bias, R, out, H, W, Cin, Cout, int(relu))
    cols = F.unfold(x.double().permute(2, 0, 1)[None], 3, padding=1)[0]                              # [(cin, ky, kx), H*W]
    wk = w.double().view(Cout, 3, 3, Cin).permute(0, 3, 1, 2).reshape(Cout, Cin * 9)
    exact = (wk @ cols).t() + bias.double()[None, :]
    if res:
        exact = exact + R.double()
    _check_exact(torch, out, exact, M, relu)


MOLD_CASES = [(640, 480, 256), (640, 480, 512), (640, 480, 1024), (1280, 720, 1024), (320, 240, 1024), (480, 640, 1024), (641, 479, 1024)]


@pytest.mark.parametrize("W,H,S", MOLD_CASES)
def test_mold_matches_rule(W, H, S):
    """mf_backbone_mold == R-MOLD (tests/heads_ref.mold_input) bit for bit over all S x S x 3 values: letter box, padding, the resized
    ring that blends with 0 outside the image, uint8 truncation, the mean pixel and the bf16 rounding"""
    import torch
    import maskfusion_b200 as mfb
    bb = mfb.Backbone(S, seed=1, stream=torch.cuda.current_stream().cuda_stream)
    L = bb.L

    class Dev:
        __cuda_array_interface__ = {"shape": (S, S, 3), "typestr": "<i2", "data": (L.mf_backbone_input_buffer(bb.h), False), "version": 2}
    try:
        for kind in ref.MOLD_KINDS:
            rgba = ref.mold_test_image(kind, W, H, seed=W * H + S)
            d = torch.from_numpy(rgba).cuda()
            assert L.mf_backbone_mold(C.c_void_p(bb.h), C.c_void_p(d.data_ptr()), W, H) == 0, L.mf_cnn_last_error().decode()
            torch.cuda.synchronize()
            got = torch.as_tensor(Dev(), device="cuda").cpu().numpy().view(np.uint16)
            want, _ = ref.mold_input(rgba, S)
            bad = np.argwhere(got != want)
            assert bad.shape[0] == 0, (kind, f"{bad.shape[0]} of {want.size} differ, first (y, x, c): {bad[:4].tolist()}")
        assert L.mf_backbone_mold(C.c_void_p(bb.h), None, 0, H) < 0 and L.mf_backbone_mold(C.c_void_p(bb.h), None, W, -1) < 0
    finally:
        bb.close()


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
