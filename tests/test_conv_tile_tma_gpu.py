"""N <= 128 conv tiles that are finished in shared memory and leave through a TMA store, their residual loaded by TMA one
tile ahead (two tile buffers per CTA).  Each case runs enough tiles that a CTA cycles both buffers several times, or puts
a tile edge where the TMA maps must clip it: a pixel count that is not a multiple of 128, a c_out = 96 slice of a wider
buffer with poison on both sides, a stride-2 patch overhanging the output.  Every case checks that the halo is still zero
and that the channels outside the slice keep their poison.  bf16 outputs use tools/probe_conv.run_case (|err| <= 2e-2 +
1e-2 |ref| against torch fp32), e4m3 outputs the L1-scaled criterion of test_fp8_gpu."""
import math
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tools"))
sys.path.insert(0, str(ROOT / "tests"))
from probe_conv import run_case  # noqa: E402
from test_fp8_gpu import E4M3, ACC_EPS, assert_codes_match, e4m3_tensor, ref_conv  # noqa: E402

pytestmark = pytest.mark.gpu

BF16_CASES = [
    # 4 x 162 x 162 pixel rows = 820 tiles: about six per CTA, both buffers three times
    dict(name="1x1_n64_160sq_many_tiles", n=4, h=160, w=160, cin=128, cout=64, k=1, s=1),
    dict(name="1x1_n32_res_160sq_many_tiles", n=4, h=160, w=160, cin=64, cout=32, k=1, s=1, res=True),
    # 15 x 19 = 285 pixel rows: the last tile is cut by the row extent
    dict(name="1x1_n32_res_rows_not_mult_128", n=1, h=13, w=17, cin=64, cout=32, k=1, s=1, res=True),
    dict(name="3x3_n64_rows_not_mult_128", n=3, h=7, w=9, cin=64, cout=64, k=3, s=1),
    # c_out 96 in a tile of 128 at channel offset 64 of a 256-channel buffer: poison below and above the slice
    dict(name="1x1_n96_res_coff_poison_many_tiles", n=4, h=40, w=40, cin=128, cout=96, k=1, s=1, res=True, out_ld=256,
         out_coff=64, out_poison=True),
    dict(name="3x3_n32_res", n=4, h=80, w=80, cin=64, cout=32, k=3, s=1, res=True),
    dict(name="3x3_n64_res_halo", n=4, h=80, w=80, cin=32, cout=64, k=3, s=1, res=True),
    dict(name="1x1_n128_res", n=4, h=80, w=80, cin=256, cout=128, k=1, s=1, res=True),
    # the residual is the output (training dgrad): each tile's residual is loaded before that tile is stored
    dict(name="1x1_n32_res_is_out", n=4, h=80, w=80, cin=64, cout=32, k=1, s=1, res=True, res_alias=True),
    dict(name="3x3_n64_res_is_out", n=4, h=80, w=80, cin=64, cout=64, k=3, s=1, res=True, res_alias=True),
    dict(name="3x3_n128_res_is_out_halo", n=2, h=160, w=160, cin=64, cout=128, k=3, s=1, res=True, res_alias=True),
    # stride 2: patches overhanging the 13 x 15 and 20 x 22 outputs
    dict(name="s2_n128_patch_overhang", n=2, h=26, w=30, cin=64, cout=128, k=3, s=2),
    dict(name="s2_n64_patch_overhang_res", n=2, h=40, w=44, cin=64, cout=64, k=3, s=2, res=True),
    dict(name="s2_n64_xpair_many_tiles", n=4, h=320, w=320, cin=32, cout=64, k=3, s=2, xpair=True),
    dict(name="s2_n96_coff_poison", n=2, h=26, w=30, cin=64, cout=96, k=3, s=2, out_ld=256, out_coff=128, out_poison=True),
]


@pytest.mark.parametrize("case", BF16_CASES, ids=[c["name"] for c in BF16_CASES])
def test_tile_tma_bf16(case):
    r = run_case(case)
    assert r["err_word"] == 0 and r["nan"] == 0
    assert r["halo_ok"], "kernel wrote into the halo or outside its channel slice"
    assert r["ok"], r


E4M3_CASES = [
    dict(name="1x1_n32_many_tiles", n=4, h=80, w=80, ci=64, co=32, k=1, s=1),
    dict(name="1x1_n32_res_many_tiles", n=4, h=80, w=80, ci=64, co=32, k=1, s=1, res=True),
    dict(name="3x3_n64", n=2, h=40, w=40, ci=64, co=64, k=3, s=1),
    dict(name="3x3_n64_res", n=2, h=40, w=40, ci=64, co=64, k=3, s=1, res=True),
    dict(name="1x1_n128_concat", n=2, h=40, w=40, ci=256, co=128, k=1, s=1, out_ld=384, out_coff=128),
    dict(name="1x1_n128_res", n=2, h=40, w=40, ci=256, co=128, k=1, s=1, res=True),
    dict(name="1x1_n96_res_coff_rows_not_mult_128", n=1, h=13, w=17, ci=64, co=96, k=1, s=1, res=True, out_ld=256,
         out_coff=64),
    dict(name="3x3s2_n128_patch_overhang_res", n=2, h=26, w=30, ci=64, co=128, k=3, s=2, res=True),
    dict(name="bf16in_3x3s1_n64", n=2, h=40, w=40, ci=32, co=64, k=3, s=1, bf16_in=True),
]


@pytest.mark.parametrize("case", E4M3_CASES, ids=[c["name"] for c in E4M3_CASES])
def test_tile_tma_e4m3(case):
    from yolov3_b200 import ops
    from yolov3_b200.tensors import PaddedNHWC

    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(17)
    n, h, w, ci, co, k, s = (case[x] for x in ("n", "h", "w", "ci", "co", "k", "s"))
    s_in, s_out = 0.011, 0.023
    if case.get("bf16_in"):
        x = PaddedNHWC.zeros(n, h, w, ci, ld=ci + 16).slice(16, ci).load_nchw(torch.randn(n, ci, h, w, generator=g).cuda())
    else:
        x = e4m3_tensor(n, h, w, ci, ci + 32, 16, s_in, g)
    wt = torch.randn(co, ci, k, k, generator=g) / math.sqrt(ci * k * k)
    b = torch.randn(co, generator=g) * 0.1
    if case.get("bf16_in"):
        wq, bq = ops.pack_conv_weight(wt, b)
        dq = None
        wd = wq[:co].float().view(co, k, k, ci).permute(0, 3, 1, 2)
    else:
        wq, bq, sw = ops.pack_conv_weight_e4m3(wt, b)
        dq = (sw * x.scale).contiguous()
        wd = (wq.float() * sw[:, None])[:co].view(co, k, k, ci).permute(0, 3, 1, 2)
    ho, wo = h // s, w // s
    out_ld, out_coff = case.get("out_ld", co), case.get("out_coff", 0)
    ob = torch.zeros(n, ho + 2, wo + 2, out_ld, dtype=E4M3, device="cuda")
    ob.view(torch.uint8)[:, 1:-1, 1:-1] = torch.randint(0, 0x7E, (n, ho, wo, out_ld), generator=g, dtype=torch.uint8).cuda()
    before = ob.clone()
    out = PaddedNHWC(ob, out_coff, co, s_out)
    res = e4m3_tensor(n, ho, wo, co, co + 16, 16, 0.017, g) if case.get("res") else None
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.conv_bn_act(x, wq, bq, co, k, s, ops.ACT_SILU, out=out, res=res, dq=dq, err=err)
    torch.cuda.synchronize()
    assert int(err.item()) == 0
    ref, l1 = ref_conv(x.values(), wd, b.cuda(), s, True, res.values() if res is not None else None, l1=True)
    if case.get("bf16_in"):  # bf16 operands: the MMA accumulates in fp32 (summation order only)
        l1 = l1 * (2.0 ** -13 / ACC_EPS)
    assert_codes_match(ob[:, 1:-1, 1:-1, out_coff:out_coff + co], ref / s_out, l1 / s_out, case["name"])
    # the halo is still zero and the other channels keep their poison
    mask = torch.ones(ob.shape, dtype=torch.bool, device="cuda")
    mask[:, 1:-1, 1:-1, out_coff:out_coff + co] = False
    assert torch.equal(ob.view(torch.uint8)[mask], before.view(torch.uint8)[mask])
