"""Sharded validation on the GPU (prints one JSON line):

* one GPU (default): the gather of per-image results after the batch loop on KAIST-shaped synthetic results (2 252 images
  of B = 1, 0-300 kept rows each, native boxes): ``icaf_val_pack`` + ``icaf_val_merge`` + the copy of the flat arrays to
  the host (``pack_merge_ms``) against test.test's per-batch ``.cpu()`` of det / count / correct / native
  (``per_batch_cpu_ms``), each the median of ``--passes`` passes, alternated;
* ``--ranks`` under ``torchrun --nproc_per_node N`` (N >= 2 GPUs): whole ``test.test`` wall time of yolov5l FLIR with
  synthetic weights, 544 x 672, B = 1, graphed, with ``compute_loss`` and ``save_txt``, sharded over the N ranks
  (``sharded_s``) against rank 0 alone (``one_rank_s``), medians of ``--passes`` alternated passes;
* the card name, power limit and max SM clock, read in the same run.

    python scripts/val_shard_times.py [--images 2252] [--passes 5]
    torchrun --nproc_per_node 8 scripts/val_shard_times.py --ranks [--images 512]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from icafusion_b200 import ops  # noqa: E402

NIOU, MAX_DET = 10, 300


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def synthetic(n_images, dev, seed=4):
    g = np.random.Generator(np.random.PCG64(seed))
    out = []
    for k in range(n_images):
        det = torch.from_numpy(g.random((1, MAX_DET, 6), dtype=np.float32)).to(dev)
        count = torch.tensor([int(g.integers(0, MAX_DET + 1))], dtype=torch.int32, device=dev)
        correct = torch.from_numpy((g.random((1, MAX_DET, NIOU)) < 0.3).astype(np.uint8)).to(dev)
        native = torch.from_numpy(g.random((1, MAX_DET, 4), dtype=np.float32) * 640).to(dev)
        out.append((det, count, correct, native, k))
    return out


def host_loop(batches):
    rows = 0
    for det, count, correct, native, _ in batches:
        d, c, k, n = det.cpu().numpy(), count.cpu().tolist(), correct.cpu().numpy().astype(bool), native.cpu().numpy()
        rows += c[0]
    return rows


def pack_merge(batches, n_images):
    buf = ops.val_pack(batches, NIOU, native=True)
    head = buf[:4].cpu().tolist()
    m = ops.val_merge(buf[None, :head[3]].contiguous(), n_images, head[1], NIOU, native=True)
    ops.val_merge_check(m["status"].cpu().tolist(), head[1])
    return [m[k].cpu().numpy() for k in ("correct", "conf", "pcls", "native", "counts", "offsets")]


def one_gpu(args):
    dev = torch.device("cuda", 0)
    batches = synthetic(args.images, dev)
    torch.cuda.synchronize()
    pack_merge(batches, args.images)
    host_loop(batches)
    t_pm, t_host = [], []
    for _ in range(args.passes):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pack_merge(batches, args.images)
        t_pm.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host_loop(batches)
        t_host.append(time.perf_counter() - t0)
    return dict(images=args.images, pack_merge_ms=1e3 * statistics.median(t_pm), per_batch_cpu_ms=1e3 * statistics.median(t_host),
                passes=args.passes)


def ranks(args):
    import torch.distributed as dist
    from icafusion_b200 import Model
    from icafusion_b200 import test as T
    from icafusion_b200.engine import ValidationGraphs
    from icafusion_b200.loss import ComputeLoss
    from icafusion_b200.synth import load_synth
    dist.init_process_group("nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    model = Model("yolov5l_Transfusion_FLIR").eval()
    load_synth(model, 3)
    model = model.to(dev)
    model.hyp, model.gr = dict(box=0.05, obj=1.0, cls=0.5, cls_pw=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0), 1.0
    g = torch.Generator().manual_seed(2)
    shape = ((512, 640), ((1.0, 1.0), (16.0, 16.0)))
    loader = []
    for k in range(args.images):
        img = (torch.rand(1, 6, 544, 672, generator=g) * 255).to(torch.uint8).pin_memory()
        tg = torch.cat([torch.zeros(10, 1), torch.randint(0, 3, (10, 1), generator=g).float(),
                        torch.rand(10, 2, generator=g) * 0.8 + 0.1, torch.rand(10, 2, generator=g) * 0.2 + 0.02], 1)
        loader.append((img, tg.pin_memory(), [f"/d/{k:05d}.jpg"], [shape]))
    kw = dict(compute_loss=ComputeLoss(model), save_txt=True, labels_list=sorted(f"{k:05d}.txt" for k in range(args.images)))
    data = {"nc": 3, "names": ["0", "1", "2"]}
    graphs = ValidationGraphs(model)
    tmp = tempfile.mkdtemp()

    def sharded():
        return T.test(data, model=model, dataloader=loader, save_dir=tmp, graphs=graphs, group=dist.group.WORLD, **kw)

    def alone():
        if rank == 0:
            return T.test(data, model=model, dataloader=loader, save_dir=tmp, graphs=graphs, **kw)

    sharded()
    alone()
    t_sh, t_one = [], []
    for _ in range(args.passes):
        for fn, acc in ((sharded, t_sh), (alone, t_one)):
            dist.barrier()
            t0 = time.perf_counter()
            fn()
            dist.barrier()
            acc.append(time.perf_counter() - t0)
    out = dict(ranks=world, images=args.images, sharded_s=statistics.median(t_sh), one_rank_s=statistics.median(t_one),
               passes=args.passes)
    dist.destroy_process_group()
    return out if rank == 0 else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=None)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--ranks", action="store_true", help="whole-call timing under torchrun (needs >= 2 GPUs)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("val_shard_times.py measures on a CUDA device; none is visible")
    args.images = args.images or (512 if args.ranks else 2252)
    out = ranks(args) if args.ranks else one_gpu(args)
    if out is not None:
        out["card"] = card()
        print(json.dumps(out))


if __name__ == "__main__":
    main()
