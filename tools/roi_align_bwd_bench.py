#!/usr/bin/env python
"""Time the ROIAlign backward gather (`c3d_roi_align_bwd`) at the shapes the DLA34 train step gives it.

    python tools/roi_align_bwd_bench.py [--iters 100] [--save-rois FILE]   # kernel alone, CUDA events
    python tools/roi_align_bwd_bench.py --profile                            # top kernels of one graph-replayed step

The kernel mode builds the model at the bench.py shape (batch 32 at 640x640), runs two eager train steps and keeps the
`rois` and `dout` that `nnfunc.ROIAlign.backward` receives in the last one, plus the shapes of p2..p5.  It then times
the library call alone (gradient maps allocated once, outside the timed window) and, for comparison, the Python front
end `kernels.roi_align_bwd`, which also allocates the maps.  It prints the work the gather has to do — the number of
(RoI, bin, sample, tap) contributions, each applied to every channel, and the bytes of dout read once plus the maps
written once — and the least time those need on the card.

The profile mode takes a torch.profiler trace (CUDA activity) of one graph-replayed step in a process of its own,
since tracing slows the host, and prints the kernels with the largest total time.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_GBS = 3350.0          # H100 SXM data sheet, HBM3
FP32_TFLOPS = 67.0        # H100 SXM data sheet, dense FP32 (one FMA = 2 FLOP)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "nvidia-smi unavailable"
    return q


def make_trainer(batch, size):
    import torch
    from omni3d_b200 import cubercnn as pc
    from omni3d_b200 import synth
    from omni3d_b200.train import FlatSGDTrainer
    cfg = pc.load_cfg("cubercnn_DLA34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none", "MODEL.DEVICE", "cuda",
                                                 "SOLVER.IMS_PER_BATCH", batch, "SOLVER.BASE_LR", 0.0025])
    torch.manual_seed(0)
    model = pc.build_model(cfg)
    model.train()
    trainer = FlatSGDTrainer(cfg, model)
    items = synth.make_batch(batch, size, size, num_gt=8, seed=100, image_dtype=torch.uint8)
    items = [{**it, "image": it["image"].cuda(), "gt": {k: v.cuda() for k, v in it["gt"].items()}} for it in items]
    return trainer, items


def work(rois, C, P, level_shapes, strides):
    """(contributions, algorithmic bytes) of one backward: every valid RoI adds P*P bins x gh*gw samples x 4 taps, each to
    C channels; dout (bf16) is read once and every fp32 map element written once."""
    import numpy as np
    r = rois.double().cpu().numpy()
    ok = np.isfinite(r).all(1) & (r[:, 0] >= 0) & (r[:, 1] >= 0) & (r[:, 1] < len(level_shapes))
    lvl = np.where(ok, r[:, 1], 0).astype(np.int64)
    sc = np.array([1.0 / s for s in strides], dtype=np.float32)[lvl]
    f = r.astype(np.float32)
    sw, sh = f[:, 2] * sc - np.float32(0.5), f[:, 3] * sc - np.float32(0.5)
    rw, rh = f[:, 4] * sc - np.float32(0.5) - sw, f[:, 5] * sc - np.float32(0.5) - sh
    gh = np.ceil(rh / np.float32(P)).astype(np.int64)
    gw = np.ceil(rw / np.float32(P)).astype(np.int64)
    per = np.where(ok & (gh > 0) & (gw > 0), P * P * gh * gw * 4, 0)
    contrib = int(per.sum())
    R = rois.shape[0]
    map_bytes = sum(n * h * w * C * 4 for (n, h, w, _) in level_shapes)
    dout_bytes = R * P * P * C * 2
    return contrib, dout_bytes + map_bytes, {"rois": R, "valid_rois": int(ok.sum()),
                                              "rois_per_level": np.bincount(lvl[ok], minlength=len(level_shapes)).tolist()}


def kernel_mode(args):
    import numpy as np
    import torch
    from omni3d_b200 import _lib, nnfunc
    from omni3d_b200 import kernels as Kx
    trainer, items = make_trainer(args.batch, args.size)
    trainer.use_graph = False
    seen = {}
    orig = nnfunc.ROIAlign.backward

    def spy(ctx, dout):
        rois, *feats = ctx.saved_tensors
        seen.update(rois=rois.clone(), dout=dout.contiguous().clone(), shapes=[tuple(f.shape) for f in feats],
                    strides=list(ctx.cfg[0]), pooled=ctx.cfg[1])
        return orig(ctx, dout)

    nnfunc.ROIAlign.backward = staticmethod(spy)
    try:
        for _ in range(2):
            trainer.step(items)
        torch.cuda.synchronize()
    finally:
        nnfunc.ROIAlign.backward = staticmethod(orig)
    del trainer
    torch.cuda.empty_cache()

    rois, dout, shapes, strides, P = seen["rois"], seen["dout"], seen["shapes"], seen["strides"], seen["pooled"]
    if args.save_rois:
        os.makedirs(os.path.dirname(os.path.abspath(args.save_rois)), exist_ok=True)
        np.save(args.save_rois, rois.cpu().numpy())
    C = shapes[0][3]
    feats = [torch.empty(s, device="cuda", dtype=torch.bfloat16) for s in shapes]
    grads = [torch.zeros(s, device="cuda", dtype=torch.float32) for s in shapes]
    lv = Kx._levels(feats, strides, grads)
    L = _lib.lib()

    def call():
        _lib.check(L.c3d_roi_align_bwd(ctypes.byref(lv), _lib.ptr(rois), rois.shape[0], C, P, P, _lib.ptr(dout), _lib.stream()))

    def events(fn, n):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(n):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return {"median_ms": float(np.median(ts)), "min_ms": float(min(ts)), "max_ms": float(max(ts)),
                "p10_ms": float(np.percentile(ts, 10)), "p90_ms": float(np.percentile(ts, 90)), "launches": n}

    kern = events(call, args.iters)
    front = events(lambda: Kx.roi_align_bwd(feats, strides, rois, dout, P), max(20, args.iters // 4))
    contrib, nbytes, counts = work(rois, C, P, shapes, strides)
    t_hbm = nbytes / (HBM_GBS * 1e9) * 1e3
    t_fma = contrib * C / (FP32_TFLOPS * 1e12 / 2) * 1e3
    print(json.dumps({
        "card": card(), "kernel": "c3d_roi_align_bwd", "C": C, "pooled": P, "level_shapes": shapes, "strides": strides,
        **counts, "c3d_roi_align_bwd": kern, "kernels.roi_align_bwd (allocates the maps)": front,
        "contributions": contrib, "channel_fmas": contrib * C, "algorithmic_bytes": nbytes,
        "bound": {"hbm_ms": t_hbm, "fp32_fma_ms": t_fma, "least_ms": max(t_hbm, t_fma),
                  "bound_by": "hbm" if t_hbm >= t_fma else "fp32 fma",
                  "source": "H100 SXM data sheet: 3.35 TB/s HBM3, 67 TFLOP/s dense FP32 (not measured)"},
        "frac_of_bound": max(t_hbm, t_fma) / kern["median_ms"]}))


def profile_mode(args):
    import torch
    from torch.profiler import ProfilerActivity, profile
    trainer, items = make_trainer(args.batch, args.size)
    for _ in range(4):                     # two eager warm-up steps, the recording, one replay
        trainer.step(items)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        trainer.step(items)
        torch.cuda.synchronize()
    trace = args.trace or os.path.join(tempfile.mkdtemp(), "step.pt.trace.json")
    prof.export_chrome_trace(trace)
    rows = {}
    for e in json.load(open(trace))["traceEvents"]:
        if e.get("cat") == "kernel":
            t = rows.setdefault(e["name"], [0.0, 0])
            t[0] += e.get("dur", 0.0) / 1e3
            t[1] += 1
    total = sum(v[0] for v in rows.values())
    top = sorted(rows.items(), key=lambda kv: -kv[1][0])[:args.top]
    print(json.dumps({"card": card(), "graph_replayed": trainer.graph is not None, "kernel_ms_total": total,
                      "top": [{"kernel": k[:120], "ms": v[0], "calls": v[1], "share": v[0] / total if total else 0.0}
                              for k, v in top]}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--iters", type=int, default=100, help="timed launches (at least 50)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="trace one graph-replayed step instead")
    ap.add_argument("--top", type=int, default=25)
    ap.add_argument("--trace", metavar="FILE", help="where the profile mode writes its chrome trace (default: a temp dir)")
    ap.add_argument("--save-rois", metavar="FILE", help="also write the captured rois as .npy")
    args = ap.parse_args()
    if args.iters < 50 and not args.profile:
        ap.error("--iters must be at least 50")
    import torch
    if not torch.cuda.is_available():
        sys.exit("roi_align_bwd_bench: needs a CUDA device")
    profile_mode(args) if args.profile else kernel_mode(args)


if __name__ == "__main__":
    main()
