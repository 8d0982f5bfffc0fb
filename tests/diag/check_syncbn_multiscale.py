"""2-rank check of --sync-bn with the ranks at DIFFERENT batch shapes (--multi-scale draws a size per rank: the reference
seeds every rank differently).  Rank 0 trains on 2 images at 320x320 and rank 1 on 2 images at 640x640, both with
parallel.convert_sync_batchnorm().  The reference is the oracle's train-mode forward with nn.SyncBatchNorm's semantics:
every BatchNorm all-reduces (sum, sum of squares, pixel count) over the ranks (autograd-aware, so the backward reduces the
gradient sums too), normalises with the combined batch statistics and updates the running statistics with momentum 0.03
and the unbiased combined variance; the loss is the oracle's ComputeLoss, scaled by the world size, and the gradients are
averaged over the ranks as DDP does.  The synchronised running statistics must equal the reference's (check_syncbn.py's
bound).  The averaged gradients must match the reference's as closely as a synchronised step with both ranks at one shape
(2 x 640x640, where the pixel count is n*h*w*world as it always was) matches its reference: at random initialisation the
bf16 pipeline's gradients differ from fp32 ones by a median relative L2 of a few tenths, so that control measures the
accuracy the mixed-shape path has to keep.
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tests/diag/check_syncbn_multiscale.py
With fewer GPUs than ranks NCCL cannot run; the ranks then share the GPUs over gloo (both on cuda:0 with one GPU)."""
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))

SHAPES = [(2, 320, 320), (2, 640, 640)]  # (n, h, w) of rank 0 and rank 1
EQUAL = (2, 640, 640)  # the control: both ranks at one shape, where the pixel count is n * h * w * world as it always was


def main():
    import torch
    import torch.distributed as dist
    import torch.distributed.nn.functional as dnn
    import torch.nn.functional as F
    import yolo_oracle as O

    from yolov3_b200 import parallel
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    assert world == len(SHAPES), f"run with --nproc-per-node {len(SHAPES)}"
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]) % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl" if torch.cuda.device_count() >= world else "gloo")
    cfg = ROOT / "yolov3_b200" / "cfg" / "yolov3.yaml"
    params = O.init_params(cfg, seed=0)
    hyp = O.scaled_hyp()

    def step(n, h, w):
        """(engine loss, oracle loss, running stats worst rel diff, gradient rel-L2 median and max) of one synchronised
        step with this rank's batch at (n, h, w)."""
        x = torch.randint(0, 256, (n, 3, h, w), dtype=torch.uint8, generator=torch.Generator().manual_seed(3 + rank))
        t = O.synth_targets(n, seed=2 + rank)

        # ---- the engine: --sync-bn with this rank's shape
        m = Model(cfg, device=dev)
        m.load_state_dict(params)
        m.hyp = hyp
        parallel.convert_sync_batchnorm(m)
        m.train()
        loss, _ = ComputeLoss(m)(m(x.to(dev)), t.to(dev))
        parallel.scale_loss(loss).backward()
        P = m.device_params()
        names = sorted(k for k in P if P[k].grad is not None)
        parallel.allreduce_gradients([P[k] for k in names])
        torch.cuda.synchronize()
        got_grad = {k: P[k].grad.detach().float().cpu() for k in names}
        got_run = {k: v.detach().float().cpu() for k, v in P.items() if "running" in k}

        # ---- the reference: the oracle with nn.SyncBatchNorm's statistics over both ranks' pixels, in fp32 (no TF32)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        ref = {k: v.to(dev).float().clone() for k, v in params.items()}
        for k in names:
            ref[k].requires_grad_(True)
        running = {}

        class SyncOracle(O.OracleModel):
            def conv_block(self, xin, prefix, k, s):
                p = self.params
                y = F.conv2d(xin, p[prefix + ".conv.weight"], None, stride=s, padding=k // 2)
                c = y.shape[1]
                cnt = torch.full((1,), float(y.numel() // c), device=y.device)
                tot = dnn.all_reduce(torch.cat([y.sum((0, 2, 3)), (y * y).sum((0, 2, 3)), cnt]))
                N = tot[2 * c]
                mean = tot[:c] / N
                var = tot[c:2 * c] / N - mean * mean
                z = (y - mean.view(1, c, 1, 1)) * torch.rsqrt(var + O.BN_EPS).view(1, c, 1, 1)
                z = z * p[prefix + ".bn.weight"].view(1, c, 1, 1) + p[prefix + ".bn.bias"].view(1, c, 1, 1)
                with torch.no_grad():
                    running[prefix + ".bn.running_mean"] = 0.97 * p[prefix + ".bn.running_mean"] + 0.03 * mean
                    running[prefix + ".bn.running_var"] = 0.97 * p[prefix + ".bn.running_var"] + 0.03 * var * N / (N - 1)
                return z * torch.sigmoid(z)

        om = SyncOracle(cfg, params=ref, train=True)
        raw = om.detect_raw(om.forward_features(x.to(dev).float() / 255))
        loss_o, _ = O.compute_loss([r.cpu() for r in raw], t, params["model.28.anchors"], hyp)
        (loss_o * world).backward()
        ref_grad = {}
        for k in names:
            g = ref[k].grad.detach().clone()
            dist.all_reduce(g)
            ref_grad[k] = (g / world).float().cpu()
        ref_run = {k: v.float().cpu() for k, v in running.items()}
        assert set(ref_run) == set(got_run), sorted(set(ref_run) ^ set(got_run))
        worst = max(float((got_run[k] - ref_run[k]).abs().max() / ref_run[k].abs().max().clamp_min(1e-6)) for k in ref_run)
        errs = sorted(float((got_grad[k] - ref_grad[k]).norm() / ref_grad[k].norm().clamp_min(1e-30)) for k in names)
        return float(loss), float(loss_o), worst, errs[len(errs) // 2], errs[-1]

    n, h, w = SHAPES[rank]
    loss, loss_o, worst_rs, med, mx = step(n, h, w)
    _, _, worst_eq, med_eq, _ = step(*EQUAL)
    print(f"rank {rank} {n}x{h}x{w}: loss {loss:.4f} (oracle {loss_o:.4f}); running stats worst rel diff {worst_rs:.2e}; "
          f"gradient rel-L2 median {med:.3f} max {mx:.3f}; equal shapes {EQUAL}: running stats {worst_eq:.2e}, gradient "
          f"median {med_eq:.3f}")
    ok = torch.tensor([float(worst_rs < 2e-2 and worst_eq < 2e-2 and med <= 1.25 * med_eq + 0.05)], device=dev)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("SYNCBN_MULTISCALE_OK" if ok.item() else "SYNCBN_MULTISCALE_FAIL")
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok.item() else 1)


if __name__ == "__main__":
    main()
