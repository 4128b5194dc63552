"""Per-shape timing of the wgmma conv kernels on the layer shapes of DLA34_FPN @ 640^2, batch 32
(SURVEY.md section 8a-2 census): CUDA-event ms and algorithmic TFLOP/s for forward, data gradient and weight
gradient, with the multiplicity of every shape in one train step, so the table sums to the conv time of a step.
Also the target of the ncu --set full captures under profiles/ (ONLY=<substring> KIND=fwd|dgrad|wgrad)."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from omni3d_b200 import conv as K
from omni3d_b200 import nnfunc

STEM_C = 8     # NHWC8 image for the rolling-halo stem kernel
SHAPES = [  # name, H, W, Cin, Cout, k, stride, pad, real_cin, count in DLA34_FPN (+RPN head), has_dgrad
    ("stem7x7_3(%d)->16@640" % STEM_C, 640, 640, STEM_C, 16, 7, 1, 3, 3, 1, False),
    ("level0_16->16@640", 640, 640, 16, 16, 3, 1, 1, 16, 1, True),
    ("level1_16->32s2@640", 640, 640, 16, 32, 3, 2, 1, 16, 1, True),
    ("l2_32->64s2@320", 320, 320, 32, 64, 3, 2, 1, 32, 1, True),
    ("l2_64->64@160", 160, 160, 64, 64, 3, 1, 1, 64, 3, True),
    ("l2_root_128->64_1x1@160", 160, 160, 128, 64, 1, 1, 0, 128, 1, True),
    ("l2_proj_32->64_1x1@160", 160, 160, 32, 64, 1, 1, 0, 32, 1, True),
    ("l3_64->128s2@160", 160, 160, 64, 128, 3, 2, 1, 64, 1, True),
    ("l3_128->128@80", 80, 80, 128, 128, 3, 1, 1, 128, 7, True),
    ("l3_root_256->128_1x1@80", 80, 80, 256, 128, 1, 1, 0, 256, 1, True),
    ("l3_root_448->128_1x1@80", 80, 80, 448, 128, 1, 1, 0, 448, 1, True),
    ("l3_proj_64->128_1x1@80", 80, 80, 64, 128, 1, 1, 0, 64, 1, True),
    ("l4_128->256s2@80", 80, 80, 128, 256, 3, 2, 1, 128, 1, True),
    ("l4_256->256@40", 40, 40, 256, 256, 3, 1, 1, 256, 7, True),
    ("l4_root_512->256_1x1@40", 40, 40, 512, 256, 1, 1, 0, 512, 1, True),
    ("l4_root_896->256_1x1@40", 40, 40, 896, 256, 1, 1, 0, 896, 1, True),
    ("l4_proj_128->256_1x1@40", 40, 40, 128, 256, 1, 1, 0, 128, 1, True),
    ("l5_256->512s2@40", 40, 40, 256, 512, 3, 2, 1, 256, 1, True),
    ("l5_512->512@20", 20, 20, 512, 512, 3, 1, 1, 512, 3, True),
    ("l5_root_1280->512_1x1@20", 20, 20, 1280, 512, 1, 1, 0, 1280, 1, True),
    ("l5_proj_256->512_1x1@20", 20, 20, 256, 512, 1, 1, 0, 256, 1, True),
    ("fpn_lat_64->256_1x1@160", 160, 160, 64, 256, 1, 1, 0, 64, 1, True),
    ("fpn_lat_128->256_1x1@80", 80, 80, 128, 256, 1, 1, 0, 128, 1, True),
    ("fpn_lat_256->256_1x1@40", 40, 40, 256, 256, 1, 1, 0, 256, 1, True),
    ("fpn_lat_512->256_1x1@20", 20, 20, 512, 256, 1, 1, 0, 512, 1, True),
    ("fpn_out/rpn_256->256@160", 160, 160, 256, 256, 3, 1, 1, 256, 2, True),
    ("fpn_out/rpn_256->256@80", 80, 80, 256, 256, 3, 1, 1, 256, 2, True),
    ("fpn_out/rpn_256->256@40", 40, 40, 256, 256, 3, 1, 1, 256, 2, True),
    ("fpn_out/rpn_256->256@20", 20, 20, 256, 256, 3, 1, 1, 256, 2, True),
    ("fpn_out/rpn_256->256@10", 10, 10, 256, 256, 3, 1, 1, 256, 2, True),
    ("rpn_pred_256->16_1x1@160", 160, 160, 256, 16, 1, 1, 0, 256, 1, True),
    ("rpn_pred_256->16_1x1@80", 80, 80, 256, 16, 1, 1, 0, 256, 1, True),
]
N = int(os.environ.get("BATCH", "32"))
ITERS = int(os.environ.get("ITERS", "5"))
only = os.environ.get("ONLY")
kind = os.environ.get("KIND", "fwd,dgrad,wgrad").split(",")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")     # > 50 MB L2 (H100)


def timeit(fn):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(ITERS):
        flush.zero_()                                  # cold L2 between timed launches
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


out = []
tot = {"fwd": 0.0, "dgrad": 0.0, "wgrad": 0.0, "gflop": 0.0}
for name, H, W, Cin, Cout, k, s, p, rc, count, has_dgrad in SHAPES:
    if only and not any(o in name for o in only.split(",")):
        continue
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(N, H, W, Cin, device="cuda", generator=g).bfloat16()
    w32 = torch.nn.Parameter(torch.randn(Cout, Cin, k, k, device="cuda", generator=g) * 0.05)
    w = w32.detach().permute(0, 2, 3, 1).contiguous().bfloat16()
    Ho, Wo = K.out_hw(H, W, k, k, s, p)
    dy = torch.randn(N, Ho, Wo, Cout, device="cuda", generator=g).bfloat16()
    dw = torch.zeros(Cout, k, k, Cin, device="cuda")
    flop = 2.0 * N * Ho * Wo * Cout * k * k * rc
    rec = {"shape": name, "count": count, "gflop": flop / 1e9}
    if "fwd" in kind:
        bn_layer = not name.startswith(("fpn", "rpn"))          # backbone convs feed BatchNorm (partial statistics in the epilogue)
        bias = None if bn_layer else torch.zeros(Cout, device="cuda")
        t = timeit(lambda: K.conv2d_fwd(x, w, bias, stride=s, pad=p, want_stats=bn_layer))
        rec.update(fwd_ms=t, fwd_tflops=flop / t / 1e9); tot["fwd"] += t * count
    if "dgrad" in kind and has_dgrad:
        nnfunc._dgrad(dy, w32, s, p, (H, W))           # fills the pack caches (packing is not part of the timed launch)
        t = timeit(lambda: nnfunc._dgrad(dy, w32, s, p, (H, W)))
        rec.update(dgrad_ms=t, dgrad_tflops=flop / t / 1e9); tot["dgrad"] += t * count
    if "wgrad" in kind:
        t = timeit(lambda: K.conv2d_wgrad(x, dy, k, k, s, p, dw=dw))
        rec.update(wgrad_ms=t, wgrad_tflops=flop / t / 1e9); tot["wgrad"] += t * count
    tot["gflop"] += flop / 1e9 * count
    out.append(rec)
    print(json.dumps(rec), flush=True)
print(json.dumps({"total_ms_per_step_weighted": tot}), flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump({"rows": out, "totals": tot}, open(os.path.join(ROOT, "gpurun_out", "conv_shapes.json"), "w"), indent=1)
