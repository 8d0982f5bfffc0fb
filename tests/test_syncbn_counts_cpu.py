"""--sync-bn with ranks at different batch shapes: every BatchNorm normalises over the sum of the ranks' pixel counts, as
nn.SyncBatchNorm's all-gathered counts give it (the reference seeds each rank differently, so under --multi-scale the
ranks draw different sizes in the same step)."""
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]

WORKER = r'''
import sys, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from yolov3_b200.train import bn_counts, gather_shapes
dist.init_process_group("gloo")
r = dist.get_rank()
mine = [(2, 320, 320), (3, 640, 480)][r]
shapes = gather_shapes(*mine)
assert shapes == [(2, 320, 320), (3, 640, 480)], shapes
n, h, w = mine
strides = [1, 2, 4, 8, 16, 32, 16, 8]                   # down the backbone, then up through the two Upsample layers
grids = [(h // s, w // s) for s in strides]
got = bn_counts(shapes, h, w, grids)
want = [float(2 * (320 // s) * (320 // s) + 3 * (640 // s) * (480 // s)) for s in strides]
assert got == want, (got, want)
same = bn_counts([mine, mine], h, w, grids)            # equal shapes: count * world, as before
assert same == [float(2 * n * gh * gw) for gh, gw in grids], same
sys.stdout.write(f"COUNTS_OK {r}\n")  # one write: the ranks share the pipe, and print's pieces interleave
sys.stdout.flush()
dist.barrier(); dist.destroy_process_group()
'''


def test_sync_bn_counts_sum_the_ranks_pixels_gloo(tmp_path):
    script = tmp_path / "counts.py"
    script.write_text(WORKER)
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
                        "127.0.0.1", "--master-port", "29655", str(script), str(ROOT)], capture_output=True, text=True,
                       timeout=240, env=dict(os.environ, MASTER_ADDR="127.0.0.1"))
    assert p.returncode == 0, p.stderr[-2000:]
    assert "COUNTS_OK 0" in p.stdout and "COUNTS_OK 1" in p.stdout
