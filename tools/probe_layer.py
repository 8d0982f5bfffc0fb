"""Run ONE conv layer shape of the yolov3 graph repeatedly (ncu target / kernel timing).

  python tools/probe_layer.py --cin 32 --cout 64 --k 3 --s 2 --hw 640 --n 32 [--res] [--iters 5] [--time]

With --time prints the CUDA-event average over the iterations (inputs of the big early layers exceed L2 on their own)."""
import argparse
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cin", type=int, required=True)
    ap.add_argument("--cout", type=int, required=True)
    ap.add_argument("--k", type=int, default=3)
    ap.add_argument("--s", type=int, default=1)
    ap.add_argument("--hw", type=int, required=True)
    ap.add_argument("--n", type=int, default=32)
    ap.add_argument("--res", action="store_true")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--time", action="store_true")
    a = ap.parse_args()

    import torch

    from yolov3_b200 import ops
    from yolov3_b200.tensors import PaddedNHWC

    g = torch.Generator().manual_seed(0)
    x = PaddedNHWC.zeros(a.n, a.hw, a.hw, a.cin)
    x.buf[:, 1:-1, 1:-1, :] = torch.randn(a.n, a.hw, a.hw, a.cin, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(a.cout, a.cin, a.k, a.k, generator=g) / (a.cin * a.k * a.k) ** 0.5
    wp, bp = ops.pack_conv_weight(w, torch.zeros(a.cout))
    ho = a.hw // a.s
    out = PaddedNHWC.zeros(a.n, ho, ho, a.cout)
    res = None
    if a.res:
        res = PaddedNHWC.zeros(a.n, ho, ho, a.cout)
        res.buf[:, 1:-1, 1:-1, :] = 1.0
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for it in range(a.iters + 2):
        if it == 2:
            ev[0].record()
        ops.conv_bn_act(x, wp, bp, a.cout, a.k, a.s, ops.ACT_SILU, out=out, res=res, err=err)
    ev[1].record()
    torch.cuda.synchronize()
    assert int(err.item()) == 0, f"watchdog code {int(err.item())}"
    if a.time:
        ms = ev[0].elapsed_time(ev[1]) / a.iters
        fl = 2.0 * a.n * ho * ho * a.cout * a.cin * a.k * a.k
        print(f"{a.cin}->{a.cout} k{a.k} s{a.s} @{a.hw} n{a.n}{' +res' if a.res else ''}: {ms * 1e3:.1f} us  {fl / ms / 1e9:.0f} TF/s")


if __name__ == "__main__":
    main()
