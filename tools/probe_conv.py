"""GPU probe: run the wgmma conv kernel over a battery of shapes and compare with torch fp32 conv2d on the same
bf16-rounded operands.  Each case runs in its own subprocess under a timeout so that a trap in one case cannot take
the others down.  Usage: python tools/probe_conv.py [--out FILE.jsonl] [case_index]  (default: probe_conv.jsonl in the system temp directory)"""
import json
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

CASES = [
    # name, n, h, w, cin, cout, k, s, extras
    dict(name="1x1_k64_n32", n=2, h=8, w=8, cin=64, cout=32, k=1, s=1),
    dict(name="1x1_k64_n64", n=1, h=10, w=14, cin=64, cout=64, k=1, s=1),
    dict(name="1x1_k128_n128", n=2, h=16, w=16, cin=128, cout=128, k=1, s=1),
    dict(name="1x1_k256_n256", n=2, h=20, w=20, cin=256, cout=256, k=1, s=1),
    dict(name="1x1_k32", n=1, h=12, w=12, cin=32, cout=64, k=1, s=1),
    dict(name="1x1_k16", n=1, h=12, w=12, cin=16, cout=32, k=1, s=1),
    dict(name="3x3_k64_n128", n=2, h=12, w=20, cin=64, cout=128, k=3, s=1),
    dict(name="3x3_k32_n64", n=1, h=16, w=16, cin=32, cout=64, k=3, s=1),
    dict(name="3x3_k16_n32", n=1, h=16, w=16, cin=16, cout=32, k=3, s=1),
    dict(name="3x3_k128_n256", n=2, h=20, w=20, cin=128, cout=256, k=3, s=1),
    dict(name="3x3_k256_n512", n=1, h=20, w=20, cin=256, cout=512, k=3, s=1),
    dict(name="3x3_k512_n1024_many_tiles", n=4, h=20, w=20, cin=512, cout=1024, k=3, s=1),
    dict(name="1x1_res", n=2, h=12, w=12, cin=64, cout=128, k=1, s=1, res=True),
    dict(name="3x3_res", n=2, h=12, w=12, cin=64, cout=128, k=3, s=1, res=True),
    dict(name="1x1_up_concat", n=2, h=10, w=10, cin=128, cout=64, k=1, s=1, upsample=True, out_ld=192, out_coff=0),
    dict(name="3x3_out_coff", n=1, h=12, w=12, cin=64, cout=64, k=3, s=1, out_ld=192, out_coff=128),
    dict(name="1x1_in_coff", n=1, h=12, w=12, cin=64, cout=64, k=1, s=1, in_ld=192, in_coff=128),
    dict(name="3x3_no_act", n=1, h=8, w=8, cin=64, cout=64, k=3, s=1, act=0),
    dict(name="s2_k64", n=2, h=16, w=16, cin=64, cout=128, k=3, s=2),
    dict(name="s2_k32", n=1, h=32, w=32, cin=32, cout=64, k=3, s=2),
    dict(name="s2_40to20", n=2, h=40, w=40, cin=128, cout=256, k=3, s=2),
    dict(name="s2_rect", n=1, h=24, w=40, cin=64, cout=64, k=3, s=2),
    dict(name="s2_wide", n=1, h=8, w=320, cin=64, cout=64, k=3, s=2),
    dict(name="s2_in_coff", n=1, h=16, w=16, cin=64, cout=64, k=3, s=2, in_ld=128, in_coff=64),
    dict(name="head_255", n=2, h=10, w=10, cin=256, cout=255, k=1, s=1, head=True, act=0),
    dict(name="head_255_k1024", n=1, h=6, w=6, cin=1024, cout=255, k=1, s=1, head=True, act=0),
    dict(name="big_flat", n=8, h=80, w=80, cin=128, cout=256, k=3, s=1),
    dict(name="s2_k32_xpair", n=2, h=32, w=48, cin=32, cout=64, k=3, s=2, xpair=True),
    dict(name="s2_k16_xpair", n=1, h=16, w=16, cin=16, cout=32, k=3, s=2, xpair=True),
    dict(name="s2_k32_xpair_many_tiles", n=4, h=160, w=160, cin=32, cout=64, k=3, s=2, xpair=True),
    dict(name="3x3_k32_res_many_tiles", n=4, h=80, w=80, cin=32, cout=64, k=3, s=1, res=True),
    dict(name="1x1_res_many_tiles", n=4, h=80, w=80, cin=128, cout=128, k=1, s=1, res=True),
    dict(name="3x3_k64_n32_res", n=2, h=40, w=40, cin=64, cout=32, k=3, s=1, res=True, act=0),   # dgrad of a 32->64 conv
    dict(name="1x1_n32_res_many_tiles", n=4, h=80, w=80, cin=64, cout=32, k=1, s=1, res=True),
    dict(name="1x1_k512_n256_res", n=2, h=40, w=40, cin=512, cout=256, k=1, s=1, res=True),      # staged, one buffer
    dict(name="3x3_k64_n64_res_many_tiles", n=4, h=80, w=80, cin=64, cout=64, k=3, s=1, res=True),
]


def run_case(c):
    import torch
    import torch.nn.functional as F

    from yolov3_b200 import ops
    from yolov3_b200.tensors import PaddedNHWC

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = "cuda"
    g = torch.Generator().manual_seed(1234)
    n, h, w, cin, cout, k, s = (c[x] for x in ("n", "h", "w", "cin", "cout", "k", "s"))
    act = c.get("act", 1)
    x = (torch.randn(n, cin, h, w, generator=g)).bfloat16().float()
    wt = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).bfloat16().float()
    b = torch.randn(cout, generator=g) * 0.5
    xin = PaddedNHWC.zeros(n, h, w, cin, ld=c.get("in_ld", cin))
    # poison the other channels of a wider buffer to catch wrong offsets
    if c.get("in_ld"):
        xin.buf[:, 1:-1, 1:-1, :] = 7.0
    xin = xin.slice(c.get("in_coff", 0), cin) if c.get("in_ld") else xin
    xin.load_nchw(x.to(dev))
    wp, bp = ops.pack_conv_weight_xpair(wt, b) if c.get("xpair") else ops.pack_conv_weight(wt, b)
    layout = 1 if c.get("xpair") else 0
    ho, wo = h // s, w // s
    u = 2 if c.get("upsample") else 1
    res = None
    res_t = None
    if c.get("res"):
        res_t = torch.randn(n, cout, ho, wo, generator=g).bfloat16().float()
        res = PaddedNHWC.zeros(n, ho, wo, cout).load_nchw(res_t.to(dev))
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    ref = F.conv2d(x.to(dev), wt.to(dev), b.to(dev), stride=s, padding=k // 2)
    if act:
        ref = ref * torch.sigmoid(ref)
    if res_t is not None:
        ref = ref + res_t.to(dev)
    if c.get("head"):
        ld = ops.cout_pad(cout)
        head = torch.full((n * ho * wo, ld), float("nan"), device=dev)
        ops.conv_bn_act(xin, wp, bp, cout, k, s, act, out_f32=head, err=err)
        torch.cuda.synchronize()
        got = head.view(n, ho, wo, ld)[..., :cout].permute(0, 3, 1, 2).contiguous()
        halo_ok = bool((head[:, cout:] == 0).all())
    else:
        out = PaddedNHWC.zeros(n, ho * u, wo * u, cout, ld=c.get("out_ld", cout))
        out = out.slice(c.get("out_coff", 0), cout) if c.get("out_ld") else out
        ops.conv_bn_act(xin, wp, bp, cout, k, s, act, out=out, res=res, upsample=bool(c.get("upsample")), err=err,
                        weight_layout=layout)
        torch.cuda.synchronize()
        got = out.to_nchw()
        if u == 2:
            ref = F.interpolate(ref, scale_factor=2, mode="nearest")
        bufc = out.buf.float()
        halo = bufc.clone()
        halo[:, 1:-1, 1:-1, :] = 0
        other = bufc[:, 1:-1, 1:-1, :].clone()
        other[..., out.coff:out.coff + cout] = 0
        halo_ok = bool((halo == 0).all()) and bool((other == 0).all())
    diff = (got - ref).abs()
    tol = 2e-2 + 1e-2 * ref.abs()
    bad = diff > tol
    res_d = dict(name=c["name"], ok=bool(not bad.any()) and halo_ok, max_abs=float(diff.max()), ref_absmax=float(ref.abs().max()),
                 n_bad=int(bad.sum()), numel=bad.numel(), halo_ok=halo_ok, err_word=int(err.item()),
                 nan=int(torch.isnan(got).sum()))
    if bad.any():
        idx = bad.nonzero()[:8].tolist()
        res_d["bad_idx"] = idx
        res_d["bad_vals"] = [(float(got[tuple(i)]), float(ref[tuple(i)])) for i in idx]
        # error pattern summaries: per-channel and per-row fractions
        res_d["bad_per_channel_nonzero"] = int((bad.sum((0, 2, 3)) > 0).sum())
        res_d["bad_rows_nonzero"] = int((bad.sum((0, 1, 3)) > 0).sum())
    # timing (rough)
    if c.get("time"):
        pass
    return res_d


def main():
    out = Path(tempfile.gettempdir()) / "probe_conv.jsonl"
    args = sys.argv[1:]
    if "--out" in args:
        out = Path(args[args.index("--out") + 1])
    if args and args[0] == "--from":  # worker: run cases [i, end) in this process, one RESULT line each
        for i in range(int(args[1]), len(CASES)):
            print(f"START {i}", flush=True)
            print("RESULT " + json.dumps(run_case(CASES[i])), flush=True)
        return
    out.parent.mkdir(parents=True, exist_ok=True)
    results = {}
    nxt = 0
    while nxt < len(CASES):
        try:
            p = subprocess.run([sys.executable, __file__, "--from", str(nxt)], capture_output=True, text=True, timeout=600)
            stdout, rc, stderr = p.stdout, p.returncode, p.stderr
        except subprocess.TimeoutExpired as e:
            stdout, rc, stderr = (e.stdout or b"").decode() if isinstance(e.stdout, bytes) else (e.stdout or ""), -9, "timeout"
        started = nxt - 1
        for l in stdout.splitlines():
            if l.startswith("START "):
                started = int(l[6:])
            elif l.startswith("RESULT "):
                results[started] = json.loads(l[7:])
        if started >= nxt and started not in results:  # the worker died inside case `started`
            results[started] = dict(name=CASES[started]["name"], ok=False, crashed=True, rc=rc, stderr=stderr[-1200:])
        nxt = max(started, nxt) + 1
    n_ok = 0
    with open(out, "w") as f:
        for i in range(len(CASES)):
            r = results.get(i, dict(name=CASES[i]["name"], ok=False, missing=True))
            n_ok += bool(r.get("ok"))
            f.write(json.dumps(r) + "\n")
            print(json.dumps(r)[:600], flush=True)
    print(f"probe_conv: {n_ok}/{len(CASES)} ok")


if __name__ == "__main__":
    main()
