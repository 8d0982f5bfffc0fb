"""Workloads of the BASELINE configs other than the headline (config 2), shared by bench.py's extra keys and the tools:

  train_step_workload   config 4: train.py-equivalent step, per-rank batch, DDP over NCCL, bf16 storage (train.py:380-421)
  spp_nms_workload      config 3: yolov3-spp forward + decode + NMS(0.25/0.45/1000), batch-sharded (detect.py:185-200)
  nms_sweep_workload    config 5: non_max_suppression on synthetic [bs,25200,85], 5 thresholds x single/multi-label
All timings: CUDA events on the current stream, max over ranks (the caller passes ``aggregate``).
"""
from __future__ import annotations

import json
import os
import sys
import time
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

CONV_GFLOP_PER_IMG = {"yolov3.yaml": 155.891, "yolov3-spp.yaml": 156.730, "yolov3-tiny.yaml": 13.172}  # @640 (BASELINE.md §2)
TRAIN_GFLOP_PER_IMG = 3 * 155.891  # forward + dgrad + wgrad (SURVEY §8d)


def _max_over_ranks(ms: float, dev) -> float:
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return ms
    t = torch.tensor([ms], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def peaks():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.loads(p.read_text())
        return dict(hbm=d["hbm_gbs"], tf_burst=d["bf16_tflops"], tf_sustained=d.get("bf16_tflops_sustained", d["bf16_tflops"]),
                    source="measured (MEASURED_PEAKS.json), sustained bf16")
    # NVIDIA's H100 SXM data sheet (700 W card): HBM3 3.35 TB/s, dense bf16 989 TFLOP/s — not measured
    return dict(hbm=3350.0, tf_burst=989.0, tf_sustained=989.0, source="H100 SXM data sheet (dense bf16, not measured)")


# ----------------------------------------------------------------------------------------------------------------- config 4
def train_step_workload(dev, rank, world, bs=8, img=640, steps=5, warmup=3, cfg="yolov3.yaml", use_graphs=True,
                        torch_optim=False):
    """One optimizer step per iteration (accumulate = 1): host uint8 images -> H2D -> train-mode forward (im/255 fused) ->
    ComputeLoss -> loss *= WORLD_SIZE -> backward with the bucketed all-reduce overlapped -> clip(10) + SGD-nesterov + EMA ->
    loss_items read back on rank 0 (the reference formats them into its progress bar every iteration, train.py:425-431)."""
    from yolov3_b200 import parallel, synth
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model
    from yolov3_b200.optim import SGD, ModelEMA
    from yolov3_b200.train import TrainEngine

    TrainEngine.use_graphs = use_graphs
    torch.manual_seed(0)
    m = Model(cfg, device=dev)
    m.hyp = synth.scaled_hyp()
    m.train()
    ddp = parallel.DDP(m)
    ema = ModelEMA(m) if rank == 0 else None  # train.py:252: EMA on rank -1/0 only
    if torch_optim:
        opt = torch.optim.SGD(list(m.parameters()), lr=0.01, momentum=0.937, nesterov=True)
    else:
        opt = SGD(m, lr=0.01, momentum=0.937, weight_decay=5e-4, nesterov=True, max_norm=10.0, ema=ema)
    loss_fn = ComputeLoss(m)
    host = torch.randint(0, 256, (bs, 3, img, img), dtype=torch.uint8, generator=torch.Generator().manual_seed(11 + rank)).pin_memory()
    targets = synth.synth_targets(bs, seed=2 + rank).to(dev)
    items_host = torch.zeros(3).pin_memory()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    names = ["h2d", "forward", "loss", "backward_with_exchange", "optimizer_clip_ema"]
    acc = [0.0] * 5
    total_ms = 0.0

    def one_step(record=True, sync_exchange=True):
        nonlocal total_ms
        ev[0].record()
        x = host.to(dev, non_blocking=True)
        ev[1].record()
        pred = m(x)
        ev[2].record()
        loss, items = loss_fn(pred, targets)
        loss = parallel.scale_loss(loss)
        ev[3].record()
        if sync_exchange:
            loss.backward()
        else:
            with ddp.no_sync():
                loss.backward()
        ev[4].record()
        if torch_optim:
            ddp.finish()
            opt.step()
            opt.zero_grad(set_to_none=True)
        else:
            opt.step()
            opt.zero_grad()
        items_host.copy_(items, non_blocking=True)
        ev[5].record()
        torch.cuda.synchronize()
        if record:
            for k in range(5):
                acc[k] += ev[k].elapsed_time(ev[k + 1])
            total_ms += ev[0].elapsed_time(ev[5])
        return float(loss.detach()), ev[3].elapsed_time(ev[4])

    for _ in range(max(warmup, 3)):
        loss_v, _ = one_step(record=False)
    if world > 1:
        dist.barrier()
    for _ in range(steps):
        loss_v, _ = one_step()
    ms_step = _max_over_ranks(total_ms / steps, dev)
    split = {n: round(v / steps, 3) for n, v in zip(names, acc)}
    # backward without the exchange (DDP.no_sync) on the same engine: the difference is the EXPOSED part of the all-reduce
    bwd_plain = 0.0
    if world > 1:
        for _ in range(2):
            one_step(record=False, sync_exchange=False)
        t = [one_step(record=False, sync_exchange=False)[1] for _ in range(steps)]
        bwd_plain = sum(t) / len(t)
        split["backward_without_exchange"] = round(bwd_plain, 3)
        split["exposed_allreduce"] = round(max(0.0, split["backward_with_exchange"] - bwd_plain), 3)
    te = next(iter(m._train_engines.values()))
    te.check_errors()
    img_s = world * bs / (ms_step / 1e3)
    pk = peaks()
    st = m.store()
    return {
        "metric": "train images/sec @640 YOLOv3 (H2D + fwd + loss + bwd/all-reduce + clip/SGD/EMA)", "value": img_s,
        "unit": "images/s", "n_gpus": world, "batch_per_gpu": bs, "global_batch": bs * world, "ms_per_step": ms_step,
        "split_ms": split, "loss": loss_v,
        "tensor_frac": 3 * CONV_GFLOP_PER_IMG.get(Path(str(cfg)).name, 155.891) * (img / 640) ** 2 * 1e9 * (img_s / world)
        / (pk["tf_sustained"] * 1e12),
        "allreduce": {"bytes_fp32": st.n_train * 4, "buckets_mb": [round((b - a) * 4 / 1e6, 1) for a, b in te.buckets],
                      "overlapped": True, "copies": 0},
        "optimizer": "torch.optim.SGD" if torch_optim else "fused clip_grad_norm(10)+SGD-nesterov(3 groups)+ModelEMA, 3 launches",
        "cuda_graphs": bool(use_graphs), "dtype": "bf16 storage / fp32 accumulate + fp32 masters", "cfg": cfg,
    }


# ----------------------------------------------------------------------------------------------------------------- config 3
def spp_nms_workload(dev, rank, world, bs=8, img=640, steps=20, warmup=3):
    from yolov3_b200.model import Model
    from yolov3_b200.pipeline import Pipeline

    torch.manual_seed(0)
    m = Model("yolov3-spp.yaml", device=dev)
    pipe = Pipeline(m, bs, img, img, conf_thres=0.25, iou_thres=0.45, max_det=1000)
    hosts = [torch.randint(0, 256, (bs, 3, img, img), dtype=torch.uint8, generator=torch.Generator().manual_seed(31 + i + 7 * rank))
             .pin_memory() for i in range(2)]
    for _ in pipe.stream(hosts[i & 1] for i in range(max(3, warmup))):
        pass
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    n_det = 0
    for dets in pipe.stream(hosts[i & 1] for i in range(steps)):
        n_det += sum(d.shape[0] for d in dets)
    e1.record()
    torch.cuda.synchronize()
    ms = _max_over_ranks(e0.elapsed_time(e1), dev)
    pipe.engine.check_errors()
    return {"metric": "images/sec yolov3-spp @640 forward+decode+NMS(0.25/0.45/1000), host uint8 in, boxes out", "value":
            world * bs * steps / (ms / 1e3), "unit": "images/s", "n_gpus": world, "batch_per_gpu": bs, "global_batch": bs * world,
            "ms_per_step": ms / steps, "h2d_bytes_per_step": pipe.h2d_bytes, "d2h_bytes_per_step": pipe.d2h_bytes,
            "detections_per_step": n_det / steps, "path": "Pipeline.stream (two batches in flight)"}


# ----------------------------------------------------------------------------------------------------------------- config 5
def nms_sweep_workload(dev, rank, world, bs=32, reps=10):
    from yolov3_b200.nms import nms_batched
    from yolov3_b200.synth import synth_predictions

    pred = synth_predictions(bs, n_rows=25200, nc=80, seed=3).to(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    hbm = peaks()["hbm"]
    out = {}
    for conf in (0.001, 0.01, 0.05, 0.1, 0.25):
        iou = 0.6 if conf <= 0.01 else 0.45
        for ml in (False, True):
            # size the candidate capacity like non_max_suppression's exact retry does (multi-label at low conf: > 4 per row)
            cap = None
            _, _, overflow, _ = nms_batched(pred, conf, iou, multi_label=ml, max_det=300)
            worst = int(overflow.max())
            if worst:
                cap = 1 << (worst - 1).bit_length()
            for _ in range(3):
                nms_batched(pred, conf, iou, multi_label=ml, max_det=300, cap=cap)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(reps):
                _, counts, overflow, _ = nms_batched(pred, conf, iou, multi_label=ml, max_det=300, cap=cap)
            e1.record()
            torch.cuda.synchronize()
            ms = _max_over_ranks(e0.elapsed_time(e1) / reps, dev)
            gbs = bs * 25200 * 85 * 4 / (ms / 1e3) / 1e9  # ALGORITHMIC bytes: z read once, 8.568 MB/image (SURVEY §8d)
            out[f"conf{conf}_iou{iou}_{'multi' if ml else 'single'}"] = {
                "input_boxes_per_s": world * bs * 25200 / (ms / 1e3), "ms_per_batch": ms, "hbm_gbs_per_gpu": gbs,
                "hbm_frac": gbs / hbm, "kept_per_image": float(counts.float().mean()), "overflow": int(overflow.max()), "candidate_capacity": cap or "default"}
    return out
