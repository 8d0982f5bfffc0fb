"""The cp.async-ring variant of the BatchNorm/SiLU backward passes (y3_set_bn_async, default on) against the register-staged
kernels it replaces: same inputs through both, results compared BIT FOR BIT (same work units, item order and operations) —
dy, the reduced sums and every per-block partial row.  Shapes cover rows shorter than a work unit, row tails, fewer units
than blocks, c = 16 ... 1024, the SyncBatchNorm phase split and the 2x-upsample layers (which stay on the staged kernel).
The staged kernels themselves are pinned against torch autograd in tests/test_train_layers_gpu.py.  Same code as the on-device
A/B script tests/diag/ab_shot.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rnd_act(n, h, w, c, gen, scale=1.0):
    from yolov3_b200.tensors import PaddedNHWC

    t = PaddedNHWC.zeros(n, h, w, c, device="cuda")
    t.buf[:, 1:-1, 1:-1, :] = (torch.randn(n, h, w, c, device="cuda", generator=gen) * scale).to(torch.bfloat16)
    return t


@pytest.mark.parametrize("n,h,w,c,upsample", [
    (2, 5, 7, 64, False),        # less than one unit per row, fewer units than blocks
    (3, 13, 13, 512, False),     # 832 items per row: one full + one partial unit
    (2, 2, 2, 1024, False),      # the 64x64 test images' deepest layer
    (2, 32, 32, 16, False),      # yolov3-tiny's 16-channel layer
    (4, 80, 80, 256, False),     # several units per block (one wave of 396 blocks)
    (2, 160, 160, 64, False),
    (2, 20, 20, 256, True),      # 2x-upsample layer: both settings run the staged kernel
])
def test_ring_variant_is_bit_identical(n, h, w, c, upsample):
    from yolov3_b200 import _lib, train_ops
    from yolov3_b200.tensors import PaddedNHWC

    L = _lib.lib()
    gen = torch.Generator(device="cuda").manual_seed(n * 1000 + h + c)
    us = 2 if upsample else 1
    y, da = _rnd_act(n, h, w, c, gen, 2.0), _rnd_act(n, h * us, w * us, c, gen)
    st = dict(scale=torch.rand(c, device="cuda", generator=gen) + 0.5, shift=torch.randn(c, device="cuda", generator=gen) * 0.3,
              mean=torch.randn(c, device="cuda", generator=gen) * 0.2, rstd=torch.rand(c, device="cuda", generator=gen) + 0.5)
    nblk = train_ops.partial_blocks(n, h, w, c)
    prev = L.y3_set_bn_async(0)
    try:
        got = []
        for flag in (0, 1):
            L.y3_set_bn_async(flag)
            dy = PaddedNHWC.zeros(n, h, w, c, device="cuda")
            partial, sums = torch.zeros(nblk * 2 * c, device="cuda"), torch.zeros(2 * c, device="cuda")
            dbeta, dgamma = torch.zeros(c, device="cuda"), torch.zeros(c, device="cuda")
            train_ops.bn_act_bwd(y, da, dy, st, sums, partial, dbeta, dgamma, upsample=upsample)          # phase 0: both passes
            # SyncBatchNorm split: local sums (phase 1), then dy from given global sums and count (phase 2)
            dy2 = PaddedNHWC.zeros(n, h, w, c, device="cuda")
            sums2, partial2 = torch.zeros(2 * c, device="cuda"), torch.zeros(nblk * 2 * c, device="cuda")
            train_ops.bn_act_bwd(y, da, dy2, st, sums2, partial2, None, None, upsample=upsample, phase=1)
            train_ops.bn_act_bwd(y, da, dy2, st, sums2, None, None, None, upsample=upsample, phase=2, count=2.0 * n * h * w)
            torch.cuda.synchronize()
            got.append((dy.buf.clone(), sums.clone(), partial.clone(), dbeta.clone(), dgamma.clone(), dy2.buf.clone(), sums2.clone()))
    finally:
        L.y3_set_bn_async(prev)
    names = ["dy", "sums", "partial", "dbeta", "dgamma", "dy (phase 2)", "sums (phase 1)"]
    for nm, a, b in zip(names, *got):
        assert torch.equal(a, b), f"{nm}: ring variant differs from the staged kernel (max |diff| {float((a.float() - b.float()).abs().max())})"
    dy0, sums0 = got[1][0], got[1][1]
    assert bool(torch.isfinite(dy0.float()).all()) and bool((dy0 != 0).any()) and bool((sums0 != 0).any())
    assert torch.equal(got[1][1], got[1][6])                 # phase 1 alone reduces to the same sums as phase 0
    assert bool((dy0[:, 0] == 0).all()) and bool((dy0[:, :, 0] == 0).all())  # the zero halo stays zero
