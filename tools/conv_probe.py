"""GPU bring-up probe for the wgmma conv kernels: each case runs in its own process under a
timeout (a protocol bug traps or times out without taking the other cases down)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [
    # name, N,H,W,Cin,Cout,K,stride,pad, extras
    ("g1x1_64_64", 2, 16, 16, 64, 64, 1, 1, 0, {}),
    ("g1x1_128_256", 2, 16, 16, 128, 256, 1, 1, 0, {}),
    ("c3x3_64_64", 2, 32, 32, 64, 64, 3, 1, 1, {}),
    ("c3x3_w20_512", 1, 20, 20, 512, 512, 3, 1, 1, {}),
    ("c3x3_w40_256", 2, 40, 40, 256, 256, 3, 1, 1, {}),
    ("c3x3_s2_64_128", 2, 32, 32, 64, 128, 3, 2, 1, {}),
    ("c3x3_cin16", 1, 64, 64, 16, 16, 3, 1, 1, {}),
    ("c3x3_cin32_s2", 1, 64, 64, 32, 64, 3, 2, 1, {}),
    ("c1x1_cin32", 1, 32, 32, 32, 64, 1, 1, 0, {}),
    ("c3x3_bias_relu", 2, 32, 32, 64, 64, 3, 1, 1, {"bias": 1, "relu": 1}),
    ("c1x1_up2", 2, 32, 32, 128, 256, 1, 1, 0, {"bias": 1, "up2": 1}),
    ("c3x3_add", 2, 16, 16, 64, 64, 3, 1, 1, {"add": 1}),
    ("c1x1_fp32_16", 2, 16, 16, 256, 16, 1, 1, 0, {"bias": 1, "fp32": 1}),
    ("c3x3_stats", 2, 40, 40, 64, 128, 3, 1, 1, {"stats": 1}),
    ("c7x7_rpnlike", 1, 10, 10, 256, 256, 3, 1, 1, {"relu": 1, "bias": 1}),
]


def run_case(name):
    import torch
    import torch.nn.functional as F
    from omni3d_b200 import conv
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    c = [c for c in CASES if c[0] == name][0]
    _, N, H, W, Cin, Cout, K, s, p, ex = c
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(N, H, W, Cin, device="cuda", generator=g).bfloat16()
    w = (torch.randn(Cout, K, K, Cin, device="cuda", generator=g) / (K * K * Cin) ** 0.5).bfloat16()
    bias = torch.randn(Cout, device="cuda", generator=g) if ex.get("bias") else None
    Ho, Wo = conv.out_hw(H, W, K, K, s, p)
    addend = None
    if ex.get("add"):
        addend = torch.randn(N, Ho, Wo, Cout, device="cuda", generator=g).bfloat16()
    if ex.get("up2"):
        addend = torch.randn(N, Ho // 2, Wo // 2, Cout, device="cuda", generator=g).bfloat16()
    res = conv.conv2d_fwd(x, w, bias, s, p, relu=bool(ex.get("relu")), addend=addend, up2=bool(ex.get("up2")),
                          out_fp32=bool(ex.get("fp32")), want_stats=bool(ex.get("stats")))
    y, stats = res if ex.get("stats") else (res, None)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), None, s, p)
    raw = ref.permute(0, 2, 3, 1)
    ref = raw
    if bias is not None:
        ref = ref + bias
    if addend is not None:
        a = addend.float()
        if ex.get("up2"):
            a = a.repeat_interleave(2, 1).repeat_interleave(2, 2)
        ref = ref + a
    if ex.get("relu"):
        ref = ref.clamp_min(0)
    err = (y.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    out = {"case": name, "fwd_max_abs_err": err, "ref_absmax": scale, "ok_fwd": err <= 1e-2 * scale + 1e-3}
    if stats is not None:
        ssum = stats[:, 0].sum(0); ssq = stats[:, 1].sum(0)
        e1 = (ssum - raw.sum((0, 1, 2))).abs().max().item()
        e2 = ((ssq - (raw * raw).sum((0, 1, 2))).abs() / (raw * raw).sum((0, 1, 2))).max().item()
        out.update({"stats_sum_err": e1, "stats_sq_relerr": e2, "ok_stats": e1 < 1e-2 and e2 < 1e-4})
    # weight gradient
    dy = torch.randn(N, Ho, Wo, Cout, device="cuda", generator=g).bfloat16()
    dw = conv.conv2d_wgrad(x, dy, K, K, s, p)
    torch.cuda.synchronize()
    xr = x.float().permute(0, 3, 1, 2).requires_grad_(False)
    wr = w.float().permute(0, 3, 1, 2).clone().requires_grad_(True)
    F.conv2d(xr, wr, None, s, p).backward(dy.float().permute(0, 3, 1, 2))
    dwr = wr.grad.permute(0, 2, 3, 1)
    werr = (dw - dwr).abs().max().item()
    out.update({"wgrad_max_abs_err": werr, "wgrad_absmax": dwr.abs().max().item(),
                "ok_wgrad": werr <= 2e-3 * dwr.abs().max().item() + 1e-3})
    print("RESULT " + json.dumps(out), flush=True)


def main():
    if len(sys.argv) > 1:
        run_case(sys.argv[1])
        return
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    results = []
    for c in CASES:
        try:
            r = subprocess.run([sys.executable, __file__, c[0]], capture_output=True, text=True, timeout=90)
            line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
            if line:
                results.append(json.loads(line[0][7:]))
            else:
                results.append({"case": c[0], "error": (r.stderr or r.stdout)[-600:]})
        except subprocess.TimeoutExpired:
            results.append({"case": c[0], "error": "timeout"})
        print(json.dumps(results[-1]), flush=True)
    json.dump(results, open(os.path.join(ROOT, "gpurun_out", "conv_probe.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
