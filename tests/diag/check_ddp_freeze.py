"""2-rank hardware check of the data-parallel exchange with frozen layers (train.py --freeze 10; run under torchrun, one rank
per GPU):
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tests/diag/check_ddp_freeze.py
(1) The exchanged gradient of every trainable parameter equals the mean over ranks of the rank-local gradients (taken
under ``ddp.no_sync()``).  (2) No all-reduce of the backward touches a frozen slot outside the span of the trainable ones:
with --freeze 10 the backbone's slots are the tail of the gradient buffer, so none of their bytes are sent.  (3) Two fused
optimizer steps keep the replicas bit-identical, the frozen parameters included.  With and without CUDA graphs."""
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))


def main():
    import torch
    import torch.distributed as dist
    import yolo_oracle as O

    from yolov3_b200 import parallel
    from yolov3_b200 import train as train_mod
    from yolov3_b200.loss import ComputeLoss
    from yolov3_b200.model import Model
    from yolov3_b200.optim import SGD
    from yolov3_b200.train import TrainEngine

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl")
    cfg = ROOT / "yolov3_b200" / "cfg" / "yolov3.yaml"
    sent = []  # (element offset in G, elements) of every all-reduce the backward launches
    real_all_reduce = dist.all_reduce

    class _Recorder:
        def __getattr__(self, name):
            return getattr(dist, name)

        @staticmethod
        def all_reduce(t, *a, **k):
            sent.append((t.data_ptr(), t.numel()))
            return real_all_reduce(t, *a, **k)

    train_mod.dist = _Recorder()
    ok = True
    for graphs in (False, True):
        TrainEngine.use_graphs = graphs
        TrainEngine.deterministic = True
        m = Model(cfg)
        m.load_state_dict(O.init_params(cfg, seed=rank))
        m.hyp = O.scaled_hyp()
        m.train()
        for k, v in m.named_parameters():  # train.py:217-223, --freeze 10
            v.requires_grad = not any(f"model.{i}." in k for i in range(10))
        ddp = parallel.DDP(m)
        st = m.store()
        frozen = st.frozen_now()
        x = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(10 + rank)).cuda()
        t = O.synth_targets(2, seed=20 + rank).cuda()
        loss_fn = ComputeLoss(m)

        def backward(sync):
            m.zero_grad()
            loss = parallel.scale_loss(loss_fn(m(x), t)[0])
            if sync:
                loss.backward()
            else:
                with ddp.no_sync():
                    loss.backward()
            torch.cuda.synchronize()

        for _ in range(3 if graphs else 1):  # graphs: eager warm-up, capture, replay
            backward(False)
        local = st.G.clone()
        gathered = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(gathered, local)
        want = sum(g.double() for g in gathered) / world
        sent.clear()
        for _ in range(3 if graphs else 1):
            backward(True)
        ddp.finish()
        G0 = st.G.data_ptr()
        ranges = [((p - G0) // 4, (p - G0) // 4 + n) for p, n in sent]
        tail = min(st.slots[k].offset for k in frozen)
        ok &= bool(ranges) and all(0 <= a and b <= tail for a, b in ranges)
        err = 0.0
        for k, v in m.named_parameters():
            s = st.slots[k]
            if k in frozen:
                ok &= v.grad is None
            else:
                w = want[s.offset:s.offset + s.numel]
                err = max(err, float((st.G[s.offset:s.offset + s.numel].double() - w).abs().max() / want.abs().max()))
        same = st.G.double().sum()
        lo, hi = same.clone(), same.clone()
        real_all_reduce(lo, op=dist.ReduceOp.MIN)
        real_all_reduce(hi, op=dist.ReduceOp.MAX)
        ok &= err < 1e-6 and bool(lo == hi)
        if rank == 0:
            print(f"graphs={graphs}: exchanged vs mean of local gradients: max rel err {err:.2e}; identical on all ranks: "
                  f"{bool(lo == hi)}; sent [{min(a for a, _ in ranges)}, {max(b for _, b in ranges)}) of G, frozen tail from "
                  f"{tail} ({(st.n_train - tail) * 4 / 1e6:.1f} MB not sent)")
        opt = SGD(m, lr=0.01, momentum=0.937, weight_decay=5e-4, nesterov=True, max_norm=10.0)
        for _ in range(2):
            loss, _ = loss_fn(m(x), t)
            parallel.scale_loss(loss).backward()
            opt.step()
            opt.zero_grad()
        torch.cuda.synchronize()
        chk = st.P[:st.n_train].double().sum()  # BatchNorm running statistics stay rank-local (no --sync-bn)
        lo, hi = chk.clone(), chk.clone()
        real_all_reduce(lo, op=dist.ReduceOp.MIN)
        real_all_reduce(hi, op=dist.ReduceOp.MAX)
        ok &= bool(lo == hi) and bool(torch.isfinite(chk))
        if rank == 0:
            print(f"graphs={graphs}: parameters identical on all ranks after 2 fused steps: {bool(lo == hi)}")
        del m, opt, ddp
        torch.cuda.empty_cache()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    real_all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("DDP_FREEZE_OK" if int(flag) else "DDP_FREEZE_FAIL")
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if int(flag) else 1)


if __name__ == "__main__":
    main()
