"""Latency mode across ranks (SURVEY 8e, DESIGN §6), launched under torch.distributed.run (tests/test_gpu_shard.py): one frame's
T Monte-Carlo samples are split by sivo_b200.sample_ranges(T, world); every rank builds its shard, pins the frame counter, sums
its samples' softmax on the device (run_partial) and one reduce to rank 0 adds the sums on the handle's stream.  Rank 0 finalises
and compares the maps with a whole-frame handle it runs itself on the same frame: classes equal except at pixels whose top-2
mean margin is below 1e-12 (reported), |d confidence| <= 1e-12, |d entropy| <= 1e-6 (reassociated float64 sums).

Backend: NCCL with one GPU per rank when there are at least as many devices as ranks; otherwise gloo with every rank on device 0
and the sums staged through host memory (gloo's reduce takes CPU tensors), so the whole path also runs on a single GPU."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="basic", choices=["basic", "standard"])
    ap.add_argument("--T", type=int, default=6)
    ap.add_argument("--precision", default="fp16", choices=["fp16", "fp32"])
    ap.add_argument("--frame", type=int, default=41)
    ap.add_argument("--variance", action="store_true", help="also check the latency-mode variance map")
    args = ap.parse_args()

    import torch
    import torch.distributed as dist
    from bench import CROP_X, CROP_Y, NET_H, NET_W, frames, model_cache_dir, model_files
    from sivo_b200 import BayesianSegNet, BayesianSegNetParams, sample_ranges
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    nccl = world <= torch.cuda.device_count()
    dev_index = local if nccl else 0
    torch.cuda.set_device(dev_index)
    dev = torch.device("cuda", dev_index)
    if nccl:
        dist.init_process_group("nccl", device_id=dev)
    else:
        dist.init_process_group("gloo")
    cache = model_cache_dir()
    if rank == 0:
        _, proto, model, _ = model_files(args.model, args.T, cache)
    dist.barrier()
    if rank != 0:
        _, proto, model, _ = model_files(args.model, args.T, cache)  # rewrites the same prototxt: wait before anyone parses it
    dist.barrier()
    params = BayesianSegNetParams(proto, model)

    ranges = sample_ranges(args.T, world)
    shard = BayesianSegNet(params, device=dev_index, seed=1234, T=args.T, precision=args.precision, samples=ranges[rank])
    left, _, _ = frames(1, start=3)[0]
    d_bgr = torch.from_numpy(np.ascontiguousarray(left[CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W])).to(dev)
    hw = NET_H * NET_W
    d_sum = torch.empty(hw * 16, dtype=torch.float64, device=dev)
    # a real stream as the current one: the default stream's handle is 0, which the library reads as "the handle's own stream",
    # and the reduce / host copy below would not be ordered after run_partial
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    shard.set_frame(args.frame)
    shard.run_partial(d_bgr.data_ptr(), d_sum.data_ptr(), stream.cuda_stream)

    def reduce_to_rank0(t):
        if nccl:
            dist.reduce(t, dst=0)  # enqueued behind the library's work on the current stream
        else:
            h = t.cpu()
            dist.reduce(h, dst=0)
            if rank == 0:
                t.copy_(h)

    reduce_to_rank0(d_sum)
    ok = True
    if rank == 0:
        maps = lambda: (torch.empty(hw, dtype=torch.uint8, device=dev), torch.empty(hw, dtype=torch.float64, device=dev),
                        torch.empty(hw, dtype=torch.float64, device=dev))
        s_cls, s_conf, s_ent = maps()
        shard.finalize(d_sum.data_ptr(), s_cls.data_ptr(), s_conf.data_ptr(), s_ent.data_ptr(), 0, 0, stream.cuda_stream)
        full = BayesianSegNet(params, device=dev_index, seed=1234, T=args.T, precision=args.precision)
        u_cls, u_conf, u_ent = maps()
        full.set_frame(args.frame)
        full.run_device_maps(d_bgr.data_ptr(), u_cls.data_ptr(), u_conf.data_ptr(), u_ent.data_ptr(), 0, 0, stream.cuda_stream)
        torch.cuda.synchronize(dev)
        mean = (d_sum.view(hw, 16) / args.T).cpu().numpy()
        top2 = np.sort(mean, axis=1)[:, -2:]
        tie = (top2[:, 1] - top2[:, 0]) < 1e-12
        diff = (s_cls != u_cls).cpu().numpy()
        d_conf = float((s_conf - u_conf).abs().max())
        d_ent = float((s_ent - u_ent).abs().max())
        ok = not (diff & ~tie).any() and d_conf <= 1e-12 and d_ent <= 1e-6 and float(np.abs(mean.sum(axis=1) - 1).max()) < 1e-4
        print(f"world {world} ({'nccl' if nccl else 'gloo, all ranks on device 0'}), {args.model} T={args.T} {args.precision}, "
              f"samples {ranges}: class mismatches {int(diff.sum())} (near-tie pixels {int(tie.sum())}), |d confidence| {d_conf:.1e}, "
              f"|d entropy| {d_ent:.1e}")
        print("LATENCY OK" if ok else "LATENCY FAILED")
    if args.variance:
        d_cls = s_cls if rank == 0 else torch.empty(hw, dtype=torch.uint8, device=dev)
        if nccl:
            dist.broadcast(d_cls, src=0)
        else:
            h_cls = d_cls.cpu()
            dist.broadcast(h_cls, src=0)
            d_cls.copy_(h_cls)
        d_mom = torch.empty(hw * 2, dtype=torch.float64, device=dev)
        shard.variance_partial(d_cls.data_ptr(), d_mom.data_ptr(), stream.cuda_stream)
        reduce_to_rank0(d_mom)
        if rank == 0:
            s_var, u_var = torch.empty(hw, dtype=torch.float64, device=dev), torch.empty(hw, dtype=torch.float64, device=dev)
            shard.variance_finalize(d_mom.data_ptr(), s_var.data_ptr(), stream.cuda_stream)
            full.variance_device(d_cls.data_ptr(), u_var.data_ptr(), stream.cuda_stream)
            torch.cuda.synchronize(dev)
            d_var = float((s_var - u_var).abs().max())
            ok_var = d_var <= 1e-12 and bool((s_var >= 0).all())
            print(f"variance over {world} shards: |d variance| {d_var:.1e} (whole-frame max {float(u_var.max()):.3g})")
            print("VARIANCE OK" if ok_var else "VARIANCE FAILED")
            ok = ok and ok_var
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
