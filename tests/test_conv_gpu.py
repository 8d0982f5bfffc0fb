"""wgmma implicit-GEMM conv (y3_conv_bn_act_fwd) and the layer-0 conv against torch fp32 conv2d on identical
bf16-rounded operands.  Tolerance: the output is stored as bf16 (rel 2^-9) after fp32 accumulation:
|err| <= 2e-2 + 1e-2*|ref|."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tools"))
from probe_conv import CASES, run_case  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_conv_tc(case):
    r = run_case(case)
    assert r["err_word"] == 0 and r["nan"] == 0
    assert r["halo_ok"], "kernel wrote outside its interior/channel slice"
    assert r["ok"], r


@pytest.mark.parametrize("c_out,dtype,hw", [(32, torch.float32, (40, 56)), (16, torch.float32, (40, 56)), (32, torch.uint8, (40, 56)),
                                            (32, torch.float32, (21, 300)), (32, torch.uint8, (24, 260)),  # > 1 column tile
                                            (32, torch.float32, (18, 54)), (16, torch.uint8, (18, 131))])  # W % 4 != 0: scalar staging
def test_conv_first(c_out, dtype, hw):
    import torch.nn.functional as F

    from yolov3_b200 import ops

    g = torch.Generator().manual_seed(3)
    n, (h, w) = 2, hw
    if dtype == torch.uint8:
        xi = torch.randint(0, 256, (n, 3, h, w), generator=g, dtype=torch.uint8)
        x = xi.float() / 255
    else:
        x = torch.rand(n, 3, h, w, generator=g)
        xi = x
    wt = torch.randn(c_out, 3, 3, 3, generator=g) * 0.3
    b = torch.randn(c_out, generator=g) * 0.2
    w27, bb = ops.pack_first_weight(wt, b)
    out = ops.conv_first(xi.cuda(), w27, bb, c_out, in_div=255.0 if dtype == torch.uint8 else 0.0)
    ref = F.conv2d(x.cuda(), wt.cuda(), b.cuda(), padding=1)
    ref = ref * torch.sigmoid(ref)
    got = out.to_nchw()
    assert torch.allclose(got, ref, atol=1e-2, rtol=1e-2), (got - ref).abs().max()
    halo = out.buf.float().clone()
    halo[:, 1:-1, 1:-1] = 0
    assert (halo == 0).all()


@pytest.mark.parametrize("k,s,off,oob_zero,ho", [(2, 2, 0, False, 8), (2, 1, 0, True, 16), (5, 1, -2, False, 16)])
def test_maxpool(k, s, off, oob_zero, ho):
    import torch.nn.functional as F

    from yolov3_b200 import ops
    from yolov3_b200.tensors import PaddedNHWC

    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 24, 16, 16, generator=g).bfloat16().float()
    xin = PaddedNHWC.zeros(2, 16, 16, 24, ld=40).slice(8, 24).load_nchw(x.cuda())
    out = PaddedNHWC.zeros(2, ho, ho, 24, ld=32).slice(8, 24)
    ops.maxpool(xin, out, k, s, off, oob_zero)
    if oob_zero:
        ref = F.max_pool2d(F.pad(x, [0, 1, 0, 1]), 2, 1, 0)
    elif k == 5:
        ref = F.max_pool2d(x, 5, 1, 2)
    else:
        ref = F.max_pool2d(x, 2, 2, 0)
    assert torch.equal(out.to_nchw().cpu(), ref)
