#!/usr/bin/env python
"""bench.py — headline benchmark of the accelerated Cube R-CNN hot path (BASELINE.json metric).

    python bench.py --gpus N --steps K --warmup W              # our arm (1 process per GPU; torchrun for N>1)
    python bench.py --impl reference --gpus N --steps K --warmup W   # the reference's CPU path (oracle port)
    python bench.py --steps K --dump-outputs DIR                     # + the last timed step's results as DIR/*.npy

One "step" = one full train step (H2D of the batch where applicable, forward, backward, gradient all-reduce
over NCCL for N>1, stabiliser check, fused SGD) of Cube R-CNN DLA34_FPN on a synthetic batch of 32 images
640x640 per GPU (BASELINE configs[1]; weak scaling: the global batch is 32*N).  Prints ONE JSON line on rank 0.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

UNIT = "images/s"
# per backbone: config file, metric name, algorithmic train GFLOP / image and conv-family forward GMAC / image
# (SURVEY.md section 8d / BASELINE.md section 3: bottom-up + FPN 20.913 + RPN head 20.244; 0.963 = the stem, which has no dgrad)
CONFIGS = {
    "dla34": {"file": "cubercnn_DLA34_FPN.yaml", "metric": "images/sec DLA34 Cube R-CNN train step", "name": "DLA34_FPN",
              "train_gflop": 452.0, "conv_fwd_gmac": 25.081 + 20.913 + 20.244, "baseline_cfg": "configs[1]"},
    "resnet34": {"file": "cubercnn_ResNet34_FPN.yaml", "metric": "images/sec ResNet34 Cube R-CNN train step",
                 "name": "ResNet34_FPN", "train_gflop": 3 * 2 * 80.17 - 1.9, "conv_fwd_gmac": 29.904 + 20.913 + 20.244,
                 "baseline_cfg": "configs[3]"},
}


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--batch", type=int, default=32, help="images per GPU (BASELINE configs[1]: 32)")
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--cpu-batch", type=int, default=2, help="images per CPU step (bounded sample of the workload)")
    ap.add_argument("--config", default="dla34", choices=sorted(CONFIGS), help="backbone (BASELINE configs[1] / configs[3])")
    ap.add_argument("--skip-cpu-baseline", action="store_true")
    ap.add_argument("--skip-iou", action="store_true")
    ap.add_argument("--skip-torch-baseline", action="store_true",
                    help="do not time the oracle model in stock PyTorch eager on the GPU (baseline_torch_gpu)")
    ap.add_argument("--dump-outputs", metavar="DIR",
                    help="after the timed steps, write what the last timed step computed as DIR/<name>.npy")
    return ap.parse_args()


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.rows, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "100"], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except OSError:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        self.t.join(timeout=2)
        sm = sorted(float(r[0]) for r in self.rows if r and r[0].replace(".", "").isdigit())
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) > 3 + i and r[3 + i] == "Active" for r in self.rows)]
        mx = [float(r[1]) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": reasons,
                "samples": len(sm)}


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d.get("bf16_tflops_sustained", 1404.6), d.get("hbm_gbs", 6574.1), "measured (MEASURED_PEAKS.json)"
    return 989.0, 3350.0, "H100 SXM data sheet (dense bf16, HBM3), not measured"


def _hbm_peak_gbs():
    return peaks()[1]


# ---------------------------------------------------------------------------------------------------------
def physical_cores():
    try:
        import psutil
        n = psutil.cpu_count(logical=False)
        if n:
            return int(n)
    except Exception:      # noqa: BLE001
        pass
    return os.cpu_count() or 1


def cpu_train_images_per_s(config_file, batch, size, steps, warmup, threads):
    """The reference's CPU path for this metric = the oracle port (fp32, MODEL.DEVICE=cpu) doing
    forward + backward + SGD on a bounded sample (batch `batch`) of the same synthetic workload.
    -> (images/s from the MEDIAN step, median s, min s, all step times)."""
    import statistics
    import torch
    from omni3d_b200 import synth
    from oracle import cubercnn_oracle as co
    from oracle import model_io
    from detectron2.utils.events import EventStorage
    torch.set_num_threads(threads)
    torch.manual_seed(0)
    cfg = co.load_cfg(config_file)
    model = co.build_model(cfg)
    model.train()
    params = [p for p in model.parameters() if p.requires_grad]
    opt = torch.optim.SGD(params, lr=1e-4, momentum=0.9, weight_decay=1e-4)
    items = synth.make_batch(batch, size, size, num_gt=8, seed=0)
    times = []
    with EventStorage(0):
        for it in range(warmup + steps):
            t0 = time.perf_counter()
            losses = model(model_io.to_d2_inputs(items))
            opt.zero_grad()
            sum(losses.values()).backward()
            opt.step()
            if it >= warmup:
                times.append(time.perf_counter() - t0)
    med = statistics.median(times)
    return batch / med, med, min(times), times


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    C = CONFIGS[args.config]
    cores = physical_cores()
    steps, warm = max(3, min(args.steps, 5)), max(2, min(args.warmup, 3))
    ips, med, best, times = cpu_train_images_per_s(C["file"], args.cpu_batch, args.size, steps, warm, cores)
    sample = (f"oracle port fwd+bwd+SGD, fp32, batch {args.cpu_batch} x {args.size}x{args.size}, {steps} timed steps after "
              f"{warm} warm-up, {cores} threads (= physical cores); value from the median step ({med:.2f} s, min {best:.2f} s)")
    print(json.dumps({
        "impl": "reference", "metric": C["metric"], "value": ips, "unit": UNIT, "n_gpus": args.gpus, "steps": steps,
        "warmup": warm, "ms_per_step": med * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"Cube R-CNN {C['name']} train step, synthetic {args.size}x{args.size}, CPU sample batch {args.cpu_batch}"},
        "cpu_baseline": {"value": ips, "unit": UNIT, "cores": cores, "kind": "port", "sample": sample,
                         "step_seconds": times, "value_from_min_step": args.cpu_batch / best},
        "e2e": {"value": ips, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }))


def torch_gpu_baseline(config_file, batch, size, steps=5, warmup=2):
    """SURVEY 8d 'baseline_torch_gpu': the oracle restatement of the reference graph (fp32 NCHW nn.Modules, per-image
    Python loops, detectron2 semantics) executed by stock PyTorch eager on this GPU — cuDNN / cuBLAS kernels,
    torchvision ROIAlign / NMS — doing forward + backward + SGD on the SAME batch shape.  fp32 (the reference trains in
    fp32, TF32 off) and bf16 autocast.  This is the library path our kernels have to beat on this box."""
    import statistics
    import torch
    from omni3d_b200 import synth
    from oracle import cubercnn_oracle as co
    from oracle import model_io
    from detectron2.utils.events import EventStorage
    out = {}
    items = synth.make_batch(batch, size, size, num_gt=8, seed=0)
    dev_items = [{**it, "image": it["image"].cuda(), "gt": {k: v.cuda() for k, v in it["gt"].items()}} for it in items]
    for name, autocast in (("bf16_autocast", True), ("fp32", False)):
        model = opt = None
        try:
            torch.backends.cudnn.allow_tf32 = False
            torch.backends.cuda.matmul.allow_tf32 = False
            torch.manual_seed(0)
            model = co.build_model(co.load_cfg(config_file)).cuda().train()
            params = [p for p in model.parameters() if p.requires_grad]
            opt = torch.optim.SGD(params, lr=1e-4, momentum=0.9, weight_decay=1e-4)
            ts = []
            with EventStorage(0):
                for it in range(warmup + steps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                        losses = model(model_io.to_d2_inputs(dev_items))
                    opt.zero_grad(set_to_none=True)
                    sum(losses.values()).backward()
                    opt.step()
                    e1.record()
                    torch.cuda.synchronize()
                    if it >= warmup:
                        ts.append(e0.elapsed_time(e1))
            med = statistics.median(ts)
            out[name] = {"value": batch / (med * 1e-3), "unit": UNIT, "ms_per_step": med, "ms_min": min(ts), "steps": steps,
                         "warmup": warmup}
        except Exception as e:      # noqa: BLE001 — a baseline that cannot run is reported, never fatal for the bench line
            out[name] = {"error": f"{type(e).__name__}: {e}"[:300]}
        del model, opt
        torch.cuda.empty_cache()
    out["what"] = (f"oracle restatement of the reference model, stock PyTorch {torch.__version__} eager on this GPU (cuDNN/cuBLAS/"
                   f"torchvision ops), fwd+bwd+SGD, batch {batch} x {size}x{size}, inputs resident in HBM, TF32 off")
    return out


# ---------------------------------------------------------------------------------------------------------
def _top_kernel_traffic():
    """dram__bytes_read.sum + dram__bytes_write.sum of ONE launch of the dominant conv kernel from the committed
    `ncu --set full` capture (profiles/top_kernel_traffic.json: {"bytes_per_launch": ...}); None if not captured."""
    p = os.path.join(ROOT, "profiles", "top_kernel_traffic.json")
    try:
        return json.load(open(p))["bytes_per_launch"]
    except Exception:      # noqa: BLE001
        return None


def conv_roofline(trainer, items, peak_tflops, peak_src, conv_fwd_gmac):
    """One instrumented step: CUDA events around every conv_tc launch (on the launching stream) ->
    algorithmic FLOPs / summed duration for the dominant kernel family."""
    import torch
    from omni3d_b200 import conv as K
    rec = []
    o_f, o_w = K.conv2d_fwd, K.conv2d_wgrad

    def fwd(x, w, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = o_f(x, w, *a, **k)
        e1.record()
        y = out[0] if isinstance(out, tuple) else out
        rec.append((e0, e1, 2.0 * y.shape[0] * y.shape[1] * y.shape[2] * w.shape[0] * w.shape[1] * w.shape[2] * w.shape[3], "fwd",
                    x.numel() * x.element_size() + y.shape[0] * y.shape[1] * y.shape[2] * w.shape[0] * y.element_size()
                    + w.numel() * 2))
        return out

    def wgrad(x, dy, KH, KW, stride=1, pad=0, dw=None, oihw=False):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = o_w(x, dy, KH, KW, stride, pad, dw, oihw)
        e1.record()
        rec.append((e0, e1, 2.0 * dy.shape[0] * dy.shape[1] * dy.shape[2] * dy.shape[3] * KH * KW * x.shape[3], "wgrad",
                    (x.numel() + dy.numel()) * 2 + dy.shape[3] * KH * KW * x.shape[3] * 4))
        return out

    K.conv2d_fwd, K.conv2d_wgrad = fwd, wgrad
    import omni3d_b200.nnfunc as nf
    graph_mode = trainer.use_graph
    trainer.use_graph = False          # the instrumented step runs eagerly (the timed steps replay a CUDA graph)
    try:
        for _ in range(2):             # 1st pass re-warms the caching allocator (the graph owns a private pool): an
            rec.clear()                # allocation between two events would be timed as kernel time
            trainer.step(items)
            torch.cuda.synchronize()
    finally:
        K.conv2d_fwd, K.conv2d_wgrad = o_f, o_w
        trainer.use_graph = graph_mode
    ms = sum(r[0].elapsed_time(r[1]) for r in rec)
    # ALGORITHMIC conv FLOPs of one train step (SURVEY.md 8d): bottom-up (DLA34 25.081 | ResNet34 29.904) + FPN 20.913 +
    # RPN head 20.244 GMAC/img forward; backward = dgrad (no dgrad for the 0.963-GMAC stem) + wgrad.  Executed FLOPs are higher
    # (stem Cin 3 padded to 16, zero-stuffed stride-2 dgrad) and are NOT what is credited here.
    n_img = items[0]["image"].shape[0] if hasattr(items[0]["image"], "shape") and items[0]["image"].dim() == 4 else len(items)
    fl = n_img * 2.0 * (3 * conv_fwd_gmac * 1e9 - 0.963e9)
    ach = fl / (ms * 1e-3) / 1e12 if ms > 0 else 0.0
    by = {}
    # per-launch roofline: a launch can be no faster than max(FLOPs / tensor peak, algorithmic bytes / HBM peak) — the 1x1 and
    # <= 32-channel layers of the family are HBM-bound (arithmetic intensity below the ridge peak_tflops / hbm), the 3x3 layers
    # with >= 64 channels tensor-bound; `per_launch_model` sums both against the measured time
    hbm = _hbm_peak_gbs()
    cls = {"tensor_bound": [0.0, 0.0, 0.0, 0], "hbm_bound": [0.0, 0.0, 0.0, 0]}     # ms, flops, bytes, launches
    attainable_ms = 0.0
    for a, b, f, kind, nbytes in rec:
        t = by.setdefault(kind, [0.0, 0.0, 0])
        dt = a.elapsed_time(b)
        t[0] += dt; t[1] += f; t[2] += 1
        t_tensor, t_hbm = f / (peak_tflops * 1e12) * 1e3, nbytes / (hbm * 1e9) * 1e3
        attainable_ms += max(t_tensor, t_hbm)
        c = cls["tensor_bound" if t_tensor >= t_hbm else "hbm_bound"]
        c[0] += dt; c[1] += f; c[2] += nbytes; c[3] += 1
    model = {"attainable_ms": attainable_ms, "measured_ms": ms, "frac": attainable_ms / ms if ms else 0.0, "hbm_peak_gbs": hbm,
             "tensor_bound": {"ms": cls["tensor_bound"][0], "launches": cls["tensor_bound"][3],
                              "tflops": cls["tensor_bound"][1] / (cls["tensor_bound"][0] * 1e-3) / 1e12 if cls["tensor_bound"][0] else 0.0,
                              "frac_of_tensor_peak": (cls["tensor_bound"][1] / (cls["tensor_bound"][0] * 1e-3) / 1e12 / peak_tflops)
                              if cls["tensor_bound"][0] else 0.0},
             "hbm_bound": {"ms": cls["hbm_bound"][0], "launches": cls["hbm_bound"][3],
                           "GBps": cls["hbm_bound"][2] / (cls["hbm_bound"][0] * 1e-3) / 1e9 if cls["hbm_bound"][0] else 0.0,
                           "frac_of_hbm_peak": (cls["hbm_bound"][2] / (cls["hbm_bound"][0] * 1e-3) / 1e9 / hbm)
                           if cls["hbm_bound"][0] else 0.0}}
    return {"bound": "tensor", "kernel": "conv_tc_* / conv_halo_* / conv_wgrad_tc_kernel (wgmma implicit GEMM, fwd + dgrad + wgrad)",
            "achieved": ach, "peak": peak_tflops, "unit": "TFLOP/s", "frac": ach / peak_tflops, "traffic": _top_kernel_traffic(),
            "peak_source": peak_src + ", bf16 sustained (kernel timed inside a long step)",
            "launches_per_step": len(rec), "conv_ms_per_step": ms, "algorithmic_tflop_per_step": fl / 1e12,
            "executed_tflop_per_step": sum(r[2] for r in rec) / 1e12, "per_launch_model": model,
            "breakdown": {k: {"ms": v[0], "tflops": v[1] / (v[0] * 1e-3) / 1e12 if v[0] else 0, "launches": v[2]}
                          for k, v in by.items()}}


def _ncu_iou_issue_pct():
    """issue-slot utilisation of the dense IoU kernel from the committed `ncu --set full` summary (profiles/): the number
    is evidence from a profiler run, never a timing; None when the summary file is absent."""
    p = os.path.join(ROOT, "profiles", "iou3d_ncu.json")
    try:
        return json.load(open(p))
    except Exception:      # noqa: BLE001
        return None


def iou_cpu_baseline(n=100, threads_all=None):
    """pytorch3d's serial CPU algorithm as the reference calls it (omni3d_evaluation.py:1404-1412) = oracle/iou3d_oracle.c,
    on a bounded n x n cross sample of the same box distributions: 1 thread (faithful) and all physical cores (pthreads)."""
    import boxgen
    from oracle import iou3d as oracle
    threads_all = threads_all or physical_cores()
    out = {}
    for regime, L in (("dense", 1.0), ("sparse", 10.0)):
        a = boxgen.inject_degenerate(boxgen.random_boxes(n, L, 0), 0.01, 1)[0]
        b = boxgen.random_boxes(n, L, 5)
        rec = {}
        for label, th in (("serial", 1), ("threaded", threads_all)):
            oracle.iou_box3d(a[:8], b[:8], threads=th)
            ts = []
            for _ in range(3):
                t0 = time.perf_counter()
                oracle.iou_box3d(a, b, threads=th)
                ts.append(time.perf_counter() - t0)
            ts.sort()
            rec[label] = {"pairs_per_s": n * n / ts[1], "cores": th, "seconds_median": ts[1]}
        out[regime] = rec
    out["kind"] = "port"
    out["sample"] = f"{n} x {n} cross pairs per regime, C restatement of iou_box3d_cpu (oracle/iou3d_oracle.c), median of 3"
    return out


def iou_block(peak_hbm, peak_src):
    """BASELINE configs[4]: box3d_overlap pairs/s.  Cross 1000 x 1000 (the reference API) dense / sparse, plus 1 M PAIRED
    sparse pairs — the regime where HBM is the roofline (200 algorithmic B / pair, almost every pair rejected by the
    bounding-sphere test)."""
    import numpy as np
    import torch
    import boxgen
    from omni3d_b200 import box3d

    def med_ms(fn, iters=10):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return float(np.median(ts))
    out = {}
    for regime, L in (("dense", 1.0), ("sparse", 10.0)):
        a = torch.from_numpy(boxgen.inject_degenerate(boxgen.random_boxes(1000, L, 0), 0.01, 1)[0]).cuda()
        b = torch.from_numpy(boxgen.random_boxes(1000, L, 5)).cuda()
        ms = med_ms(lambda: box3d.iou_box3d(a, b))
        out[regime] = {"pairs": 1_000_000, "ms": ms, "pairs_per_s": 1e6 / (ms * 1e-3),
                       "alg_GBps": (96 * 2000 + 8e6) / (ms * 1e-3) / 1e9}
    n = 1_000_000
    a = torch.from_numpy(boxgen.random_boxes(n, 10.0, 0)).cuda()
    b = torch.from_numpy(boxgen.random_boxes(n, 10.0, 5)).cuda()
    ms = med_ms(lambda: box3d.iou_box3d_paired(a, b), iters=5)
    gbs = 200.0 * n / (ms * 1e-3) / 1e9
    out["sparse_paired"] = {"pairs": n, "ms": ms, "pairs_per_s": n / (ms * 1e-3), "alg_GBps": gbs}
    # the HBM-bound regime of the path: pairs whose bounding spheres are disjoint (boxes spread over a 100 m cube) are decided
    # by the fused prep + filter kernel alone — 192 B of corners in, 12 B (vol, iou, face count) out per pair
    a = torch.from_numpy(boxgen.random_boxes(n, 100.0, 0)).cuda()
    b = torch.from_numpy(boxgen.random_boxes(n, 100.0, 5)).cuda()
    ms_d = med_ms(lambda: box3d.iou_box3d_paired(a, b, with_counts=True), iters=5)
    out["disjoint_paired"] = {"pairs": n, "ms": ms_d, "pairs_per_s": n / (ms_d * 1e-3), "alg_GBps": 204.0 * n / (ms_d * 1e-3) / 1e9}
    # at 1e6 pairs the call (a memset node + 3 launches, ~0.1 ms) is still shaped by launch latency; the streaming rate of the
    # kernel itself shows at 4e6 pairs (0.8 GB of corners)
    a4, b4 = torch.cat([a] * 4), torch.cat([b] * 4)
    ms_d = med_ms(lambda: box3d.iou_box3d_paired(a4, b4, with_counts=True), iters=5)
    gbs_d = 204.0 * 4 * n / (ms_d * 1e-3) / 1e9
    out["disjoint_paired_4m"] = {"pairs": 4 * n, "ms": ms_d, "pairs_per_s": 4 * n / (ms_d * 1e-3), "alg_GBps": gbs_d}
    del a4, b4
    out["roofline"] = {"bound": "hbm", "kernel": "iou3d_prep_paired_kernel (+ empty clip / overflow launches), 4e6 paired pairs with "
                                                 "disjoint bounding spheres (204 algorithmic B / pair)",
                       "achieved": gbs_d, "peak": peak_hbm, "unit": "GB/s", "frac": gbs_d / peak_hbm, "traffic": None,
                       "peak_source": peak_src + ", hbm copy",
                       "sparse_paired_note": "L = 10 pairs: about 5 percent survive the sphere test and are clipped (issue-bound "
                                             f"work): {gbs:.0f} GB/s algorithmic",
                       "dense_note": "dense (overlapping) pairs are issue-slot bound, not HBM bound (8 B / pair in cross mode): "
                                     "see `ncu` for the committed issue-slot / lane-utilisation figures",
                       "ncu": _ncu_iou_issue_pct()}
    return out


def dump_outputs(out_dir, trainer, n_sample=1 << 21):
    """What the last timed step handed its caller, for comparing two builds output for output: the step's losses
    (float64, one file per loss) and the updated parameters and momentum (float32) at a fixed, seeded sample of
    n_sample positions of the flat arena (the whole arena is larger than the 64 MB this dump may take)."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    st = trainer.status(wait=True)
    for k, v in st["losses"].items():
        np.save(os.path.join(out_dir, "loss_" + k.replace("/", "_") + ".npy"), np.array(v, dtype=np.float64))
    np.save(os.path.join(out_dir, "total_loss.npy"), np.array(st["total_loss"], dtype=np.float64))
    total = trainer.flat_p.numel()
    idx = np.sort(np.random.RandomState(0).choice(total, size=min(n_sample, total), replace=False))
    sel = torch.from_numpy(idx).to(trainer.flat_p.device)
    np.save(os.path.join(out_dir, "params_sample.npy"), trainer.flat_p[sel].float().cpu().numpy())
    np.save(os.path.join(out_dir, "momentum_sample.npy"), trainer.flat_m[sel].float().cpu().numpy())
    np.save(os.path.join(out_dir, "sample_index.npy"), idx.astype(np.float64))


def run_ours(args):
    import torch
    import torch.distributed as dist
    from omni3d_b200 import _lib, synth
    from omni3d_b200 import cubercnn as pc
    from omni3d_b200.train import FlatSGDTrainer
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = torch.device("cuda", local)
    C = CONFIGS[args.config]
    cfg = pc.load_cfg(C["file"], ["MODEL.WEIGHTS_PRETRAIN", "none", "MODEL.DEVICE", "cuda", "SOLVER.IMS_PER_BATCH", args.batch * world,
                                    "SOLVER.BASE_LR", 0.0025])
    torch.manual_seed(0)
    model = pc.build_model(cfg)
    model.train()
    trainer = FlatSGDTrainer(cfg, model)
    B, S = args.batch, args.size
    # two distinct synthetic batches, alternated so that consecutive steps never re-read the same inputs from L2
    host = [synth.make_batch(B, S, S, num_gt=8, seed=100 + rank * 7 + j, image_dtype=torch.uint8) for j in range(2)]
    for hb in host:
        for it in hb:
            it["image"] = it["image"].pin_memory()
    resident = [[{**it, "image": it["image"].to(dev), "gt": {k: v.to(dev) for k, v in it["gt"].items()}} for it in hb]
                for hb in host]
    h2d = sum(it["image"].numel() * it["image"].element_size() for it in host[0]) + sum(sum(v.numel() * v.element_size() for v in it["gt"].values())
                                                               for it in host[0])

    def timed(batches, steps, read_loss):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n0 = _lib.LAUNCHES["n"]
        e0.record()
        for i in range(steps):
            trainer.step(batches[i % 2])
            if read_loss:
                trainer.status(wait=True)          # device->host read of the step's losses (pinned, 56 bytes)
        e1.record()
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        ms = e0.elapsed_time(e1)
        if world > 1:
            t = torch.tensor([ms], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t)
        return ms, _lib.LAUNCHES["n"] - n0

    for i in range(max(args.warmup, 3)):
        trainer.step(resident[i % 2])
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    ms, launches = timed(resident, args.steps, read_loss=False)
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, trainer)
    for i in range(2):
        trainer.step(host[i % 2])
    ms_e2e, _ = timed(host, args.steps, read_loss=True)
    status = trainer.status()
    peak_tf, peak_hbm, peak_src = peaks()
    # the instrumented step runs on EVERY rank (it contains the same collectives as any other step)
    roof = conv_roofline(trainer, resident[0], peak_tf, peak_src, C["conv_fwd_gmac"])
    if world > 1:
        dist.barrier()
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    ips = B * world * args.steps / (ms * 1e-3)
    ips_e2e = B * world * args.steps / (ms_e2e * 1e-3)
    line = {
        "metric": C["metric"], "value": ips, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
        "data": "synthetic",
        "config": {"workload": f"Cube R-CNN {C['name']} train step, batch {B}/GPU synthetic {S}x{S}, K=50, G=8 GT/img "
                               f"(BASELINE {C['baseline_cfg']}; weak scaling, global batch {B * world})",
                   "parallelism": f"dp{world}", "l2": "two alternating input batches (39 MB uint8 images each) + ~10 GB of "
                                                      "activations per step: working set >> 50 MB L2",
                   "cuda_graph": bool(trainer.graph is not None),
                   "images": "uint8 (3,H,W), as cubercnn/data/dataset_mapper.py:35 emits them",
                   "train_gflop_per_image": C["train_gflop"]},
        "clocks": clocks,
        "e2e": {"value": ips_e2e, "unit": UNIT, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 56,
                "ms_per_step": ms_e2e / args.steps},
        "gpu_launches": launches,
        "step_tflops_model": ips / world * C["train_gflop"] / 1e3,
        "step_frac_of_peak": ips / world * C["train_gflop"] / 1e3 / peak_tf,
        "roofline": roof,
        "final_losses": status["losses"] if status else None,
        "iterations_skipped": status["iterations_explode"] if status else None,
    }
    if not args.skip_iou and world == 1:
        line["box3d_overlap"] = iou_block(peak_hbm, peak_src)
        if not args.skip_cpu_baseline:
            line["box3d_overlap"]["cpu_baseline"] = iou_cpu_baseline()
    if not args.skip_torch_baseline and world == 1:
        del trainer, model
        torch.cuda.empty_cache()
        line["baseline_torch_gpu"] = torch_gpu_baseline(C["file"], B, S)
        for k in ("bf16_autocast", "fp32"):
            v = line["baseline_torch_gpu"].get(k, {})
            if "value" in v:
                v["ours_over_this"] = ips / v["value"]
    if not args.skip_cpu_baseline and world == 1:
        cores = physical_cores()
        cb, med, best, times = cpu_train_images_per_s(C["file"], args.cpu_batch, S, 3, 1, cores)
        line["cpu_baseline"] = {"value": cb, "unit": UNIT, "cores": cores, "kind": "port",
                                "sample": f"oracle port fwd+bwd+SGD fp32, batch {args.cpu_batch} x {S}x{S}, 3 timed steps after 1 "
                                          f"warm-up, {cores} threads (= physical cores), value from the median step "
                                          f"({med:.1f} s; min {best:.1f} s)", "step_seconds": times}
    print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    a = parse()
    if a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)
