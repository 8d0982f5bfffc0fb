"""N = 256 conv tiles that are finished in shared memory and leave through a TMA store, their residual, bias (and an e4m3
input's dq) loaded by the bulk-copy engine beside the tile.  A bf16 tile is 64 KB and cycles through one buffer, so the
next tile's residual and bias are only loaded after the previous tile's store has read the buffer; an e4m3 tile cycles
through two.  Each case runs enough tiles that a CTA reuses its buffers many times, or puts a tile edge where the TMA maps
must clip it: a pixel count that is not a multiple of 128, c_out = 288 (a second N tile of 32 channels) in a slice of a
wider buffer with poison on both sides, a stride-2 patch overhanging the output.  The N = 256 upsample, which stores from
the registers, is checked into a Concat slice with poison.  Every case checks that the halo is still zero and that the
channels outside the slice keep their poison.  bf16 outputs use tools/probe_conv.run_case (|err| <= 2e-2 + 1e-2 |ref|
against torch fp32), e4m3 outputs the L1-scaled criterion of test_fp8_gpu."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tools"))
sys.path.insert(0, str(ROOT / "tests"))
from probe_conv import run_case  # noqa: E402
from test_conv_tile_tma_gpu import test_tile_tma_e4m3 as run_e4m3_case  # noqa: E402

pytestmark = pytest.mark.gpu

BF16_CASES = [
    # 32 x 82 x 82 pixel rows = 1681 tiles: about 13 per CTA through the one buffer
    dict(name="3x3_128to256_res_80sq_n32", n=32, h=80, w=80, cin=128, cout=256, k=3, s=1, res=True),
    dict(name="1x1_512to256_40sq_n32", n=32, h=40, w=40, cin=512, cout=256, k=1, s=1),
    # c_out 288: the second N tile holds 32 channels; channel offset 64 of a 384-channel buffer, poison on both sides
    dict(name="1x1_n288_res_coff64_of384_poison", n=4, h=40, w=40, cin=128, cout=288, k=1, s=1, res=True, out_ld=384,
         out_coff=64, out_poison=True),
    # 15 x 19 = 285 pixel rows: the last tile is cut by the row extent
    dict(name="3x3_n256_res_rows_not_mult_128", n=1, h=13, w=17, cin=128, cout=256, k=3, s=1, res=True),
    # stride 2: patches overhanging the 13 x 15 output
    dict(name="s2_64to256_patch_overhang_res", n=2, h=26, w=30, cin=64, cout=256, k=3, s=2, res=True),
    # the residual is the output (training dgrad): each tile's residual is loaded before that tile is stored
    dict(name="3x3_n256_res_is_out_80sq", n=4, h=80, w=80, cin=128, cout=256, k=3, s=1, res=True, res_alias=True),
    # layer 16: nearest-2x upsample into slice 0 of a 768-channel Concat buffer, poison in the other channels
    dict(name="1x1_n256_upsample_concat_poison", n=4, h=20, w=20, cin=512, cout=256, k=1, s=1, upsample=True, out_ld=768,
         out_coff=0, out_poison=True),
]


@pytest.mark.parametrize("case", BF16_CASES, ids=[c["name"] for c in BF16_CASES])
def test_tile_tma_n256_bf16(case):
    r = run_case(case)
    assert r["err_word"] == 0 and r["nan"] == 0
    assert r["halo_ok"], "kernel wrote into the halo or outside its channel slice"
    assert r["ok"], r


E4M3_CASES = [
    # 16 x 82 x 82 pixel rows = 841 tiles: about 6 per CTA, both buffers three times
    dict(name="1x1_256to256_res_many_tiles", n=16, h=80, w=80, ci=256, co=256, k=1, s=1, res=True),
    dict(name="3x3s2_n256_patch_overhang_res", n=2, h=26, w=30, ci=64, co=256, k=3, s=2, res=True),
    dict(name="1x1_n512_coff256_of768", n=4, h=40, w=40, ci=256, co=512, k=1, s=1, out_ld=768, out_coff=256),
    dict(name="1x1_n288_res", n=4, h=20, w=20, ci=128, co=288, k=1, s=1, res=True),
]


@pytest.mark.parametrize("case", E4M3_CASES, ids=[c["name"] for c in E4M3_CASES])
def test_tile_tma_n256_e4m3(case):
    run_e4m3_case(case)
