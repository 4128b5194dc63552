"""Train-step throughput of the Bottleneck backbones (torchvision ResNet-50 / 101, DLA-46-C, DLA-60, DLA-102, DLA-169) on
one GPU.  Prints one JSON line per backbone:

* the card's name and power limit, read by the same process just before the measurement;
* images/s and ms/step of the graph-replayed FlatSGDTrainer step (batch 32 @ 640x640, or the largest power-of-two batch
  that fits, stated in the line), after warm-up, over at least 20 timed steps (CUDA events around the whole window);
* torch.cuda.max_memory_allocated of that run;
* the same model as the fp32 oracle restatement (tests/bottleneck_oracle.py) run by stock PyTorch eager under bf16 autocast
  on the same GPU, forward + backward + SGD on the same batch shape;
* for the torchvision ResNets, the CUDA-event time of the 1x1 / stride-2 data gradients (zero_stuff2 scatter + 1x1
  convolution over the scattered map) in one eager step, the route that costs 4x the needed FLOPs.

    python tests/tools/bench_backbones.py [--types resnet50,dla60] [--batch 32] [--size 640] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bottleneck_oracle as bo  # noqa: E402
from omni3d_b200 import synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout
    name, power = [s.strip() for s in q.strip().split(",")]
    return {"name": name, "power_limit": power, "torch_name": torch.cuda.get_device_name()}


def _cfg(name, batch):
    from omni3d_b200 import cubercnn as pc
    cfg_file, opts, _ = bo.CASES[name]
    return pc.load_cfg(cfg_file, ["MODEL.WEIGHTS_PRETRAIN", "none", "MODEL.DEVICE", "cuda", "SOLVER.IMS_PER_BATCH", batch,
                                  "SOLVER.BASE_LR", 0.0025] + list(opts))


def _batches(batch, size, dev):
    out = []
    for j in range(2):          # two alternating batches, resident on the device
        hb = synth.make_batch(batch, size, size, num_gt=8, seed=100 + j, image_dtype=torch.uint8)
        out.append([{**it, "image": it["image"].to(dev), "gt": {k: v.to(dev) for k, v in it["gt"].items()}} for it in hb])
    return out


def ours(name, batch, size, steps, warmup):
    from omni3d_b200 import cubercnn as pc
    from omni3d_b200 import nnfunc
    from omni3d_b200.train import FlatSGDTrainer
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.cuda.reset_peak_memory_stats()
    cfg = _cfg(name, batch)
    torch.manual_seed(0)
    model = pc.build_model(cfg).train()
    tr = FlatSGDTrainer(cfg, model)
    data = _batches(batch, size, dev)
    for i in range(max(warmup, 3)):             # two eager steps + the captured one
        tr.step(data[i % 2])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        tr.step(data[i % 2])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    st = tr.status()
    out = {"images_per_s": batch / (ms * 1e-3), "ms_per_step": ms, "cuda_graph": tr.graph is not None,
           "max_memory_allocated_bytes": torch.cuda.max_memory_allocated(),
           "final_total_loss": st["total_loss"], "iterations_skipped": st["iterations_explode"]}
    if name.startswith("resnet"):
        # one eager step with CUDA events around every 1x1 / stride-2 data gradient (zero_stuff2 + the 1x1 conv)
        calls, orig = [], nnfunc._dgrad

        def timed_dgrad(dy, w, stride, pad, in_hw, into=None):
            if stride != 2 or w.shape[2] != 1:
                return orig(dy, w, stride, pad, in_hw, into)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            r = orig(dy, w, stride, pad, in_hw, into)
            b.record()
            calls.append((a, b, tuple(dy.shape), tuple(in_hw)))
            return r
        tr.use_graph = False
        nnfunc._dgrad = timed_dgrad
        try:
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            tr.step(data[0])
            s1.record()
            torch.cuda.synchronize()
        finally:
            nnfunc._dgrad = orig
        out["dgrad_1x1_s2_zero_stuff2"] = {
            "launch_groups": len(calls), "ms_total": sum(a.elapsed_time(b) for a, b, _, _ in calls),
            "eager_step_ms": s0.elapsed_time(s1),
            "per_call": [{"dy_nhwc": s, "dx_hw": hw, "ms": a.elapsed_time(b)} for a, b, s, hw in calls]}
    del tr, model, data
    torch.cuda.empty_cache()
    return out


def eager_bf16(name, batch, size, steps=5, warmup=2):
    """the oracle restatement in stock PyTorch eager (cuDNN / cuBLAS / torchvision ops) under bf16 autocast"""
    from detectron2.utils.events import EventStorage
    from oracle import model_io
    items = synth.make_batch(batch, size, size, num_gt=8, seed=0)
    dev_items = [{**it, "image": it["image"].cuda(), "gt": {k: v.cuda() for k, v in it["gt"].items()}} for it in items]
    model = opt = None
    try:
        torch.manual_seed(0)
        model = bo.build_model(bo.load_cfg(name)).cuda().train()
        opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=1e-4, momentum=0.9, weight_decay=1e-4)
        ts = []
        with EventStorage(0):
            for it in range(warmup + steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    losses = model(model_io.to_d2_inputs(dev_items))
                opt.zero_grad(set_to_none=True)
                sum(losses.values()).backward()
                opt.step()
                e1.record()
                torch.cuda.synchronize()
                if it >= warmup:
                    ts.append(e0.elapsed_time(e1))
        med = statistics.median(ts)
        return {"images_per_s": batch / (med * 1e-3), "ms_per_step": med, "steps": steps, "warmup": warmup,
                "torch": torch.__version__}
    except torch.OutOfMemoryError as e:
        return {"error": f"OutOfMemoryError: {e}"[:200]}
    finally:
        del model, opt
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--types", default=",".join(bo.CASES))
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-eager", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_backbones.py measures on a CUDA device; none found")
    for name in args.types.split(","):
        line = {"backbone": name, "gpu": card(), "image_size": args.size, "requested_batch": args.batch}
        batch = args.batch
        while True:
            try:
                line["ours"] = ours(name, batch, args.size, max(args.steps, 20), args.warmup)
                break
            except torch.OutOfMemoryError:
                torch.cuda.empty_cache()
                if batch == 1:
                    raise
                batch //= 2
        line["batch"] = batch
        if not args.skip_eager:
            line["eager_bf16_autocast"] = eager_bf16(name, batch, args.size)
            if "images_per_s" in line["eager_bf16_autocast"]:
                line["ours_over_eager"] = line["ours"]["images_per_s"] / line["eager_bf16_autocast"]["images_per_s"]
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
