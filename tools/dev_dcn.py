"""Development driver for the tensor-core deformable-conv kernels (run on an H100).

Every case runs in its own subprocess (a trapped kernel kills only that CUDA context) with a timeout, and appends one JSON
line to gpurun_out/dev_dcn.jsonl: max relative error of precision 1 (bf16x3) and 2 (bf16) against the fp32 FFMA path
(itself pinned to the oracle by tests/test_gpu_parity.py) for forward and every gradient, plus CUDA-event timings and the
torchvision CUDA deform_conv2d time (the reference's backend) for the cfg-5 shapes.

    python tools/dev_dcn.py --all [--filter substr]
    python tools/dev_dcn.py --case NAME
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

#        name            n  cin   cout  h    w    grp dg mod    stride timed
CASES = [
    ("s_64",             2, 64,   64,   12,  20,  1,  1, False, 1, False),
    ("s_128",            2, 128,  128,  25,  42,  1,  1, False, 1, False),
    ("s_g2_mod",         2, 128,  192,  17,  23,  2,  1, True,  1, False),
    ("s_dg2_s2",         2, 256,  256,  21,  19,  1,  2, True,  2, False),
    ("s_g4_c64",         2, 256,  256,  13,  17,  4,  1, True,  1, False),
    ("s_g32_c16",        2, 512,  512,  13,  17,  32, 1, True,  1, False),
    ("s_g32_c32",        1, 1024, 1024, 9,   11,  32, 1, False, 1, False),
    ("s_k1split",        1, 512,  512,  7,   9,   1,  1, True,  1, False),
    ("c5_128_g1",        2, 128,  128,  100, 168, 1,  1, False, 1, True),
    ("c5_256_g1",        2, 256,  256,  50,  84,  1,  1, False, 1, True),
    ("c5_512_g1",        2, 512,  512,  25,  42,  1,  1, False, 1, True),
    ("c5_512_g32",       2, 512,  512,  100, 168, 32, 1, False, 1, True),
    ("c5_1024_g32",      2, 1024, 1024, 50,  84,  32, 1, False, 1, True),
    ("c5_2048_g32",      2, 2048, 2048, 25,  42,  32, 1, False, 1, True),
    ("c5_256_g1_mod",    2, 256,  256,  50,  84,  1,  1, True,  1, True),
]


def timeit(fn, rep=10, warm=3):
    import torch

    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(rep):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / rep * 1e3  # us


def run_case(name):
    import torch

    from detectron2_b200 import ops

    (_, n, cin, cout, h, w, grp, dg, mod, stride, timed) = [c for c in CASES if c[0] == name][0]
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(cin * 7 + cout + h)
    k, p = 3, 1
    ho, wo = (h + 2 * p - k) // stride + 1, (w + 2 * p - k) // stride + 1
    x = torch.randn(n, cin, h, w, generator=g).to(dev)
    off = (torch.randn(n, 2 * dg * k * k, ho, wo, generator=g) * 2).to(dev)
    mask = torch.sigmoid(torch.randn(n, dg * k * k, ho, wo, generator=g)).to(dev) if mod else None
    wt = (torch.randn(cout, cin // grp, k, k, generator=g) * (1.0 / math.sqrt(cin // grp * 9))).to(dev)
    bias = torch.randn(cout, generator=g).to(dev) if mod else None
    go = torch.randn(n, cout, ho, wo, generator=g).to(dev)
    S, P, D = [stride, stride], [p, p], [1, 1]
    res = {"case": name, "shape": [n, cin, cout, h, w, grp, dg, int(mod), stride]}

    def fwd(prec, xx=x):
        return ops.deform_conv_op(xx, off, mask, wt, bias, S, P, D, grp, dg, prec)

    def bwd(prec, xx=x):
        return ops.deform_conv_backward_op(xx, off, mask, wt, go, S, P, D, grp, dg, bias is not None, True, True, prec)

    def rel(a, b):
        return float((a - b).abs().max() / (b.abs().max() + 1e-12))

    y0 = fwd(0)
    g0 = bwd(0)
    torch.cuda.synchronize()
    for prec in (1, 2):
        try:
            y = fwd(prec)
            torch.cuda.synchronize()
            res["fwd_err_p%d" % prec] = rel(y, y0)
        except RuntimeError as e:
            res["fwd_err_p%d" % prec] = "ERR " + str(e)[:120]
        try:
            gs = bwd(prec)
            torch.cuda.synchronize()
            for nm, a, b in zip(["gx", "goff", "gmask", "gw"], gs[:4], g0[:4]):
                if b.numel():
                    res["%s_err_p%d" % (nm, prec)] = rel(a, b)
        except RuntimeError as e:
            res["bwd_err_p%d" % prec] = "ERR " + str(e)[:120]
    # channels_last input consumed in place
    try:
        xcl = x.contiguous(memory_format=torch.channels_last)
        res["fwd_err_p1_cl"] = rel(fwd(1, xcl), y0)
        gcl = bwd(1, xcl)
        res["gx_err_p1_cl"] = rel(gcl[0], g0[0])
        res["gx_cl_is_cl"] = bool(gcl[0].is_contiguous(memory_format=torch.channels_last))
    except RuntimeError as e:
        res["cl_err"] = "ERR " + str(e)[:120]
    if timed:
        flops = 2.0 * n * cout * (cin // grp) * 9 * ho * wo
        for prec in (0, 1, 2):
            try:
                res["fwd_us_p%d" % prec] = timeit(lambda: fwd(prec))
                res["bwd_us_p%d" % prec] = timeit(lambda: bwd(prec), rep=5, warm=2)
            except RuntimeError as e:
                res["time_err_p%d" % prec] = str(e)[:120]
        res["fwd_tflops_p1"] = flops / res.get("fwd_us_p1", float("inf")) / 1e6
        try:
            import torchvision.ops as tvo

            res["tv_fwd_us"] = timeit(lambda: tvo.deform_conv2d(x, off, wt, None, S, P, D, mask), rep=5, warm=2)
            xg, og, wg = x.clone().requires_grad_(True), off.clone().requires_grad_(True), wt.clone().requires_grad_(True)

            def tvb():
                yy = tvo.deform_conv2d(xg, og, wg, None, S, P, D, mask)
                yy.backward(go)
                xg.grad = og.grad = wg.grad = None

            t_fb = timeit(tvb, rep=5, warm=2)
            res["tv_bwd_us"] = t_fb - res["tv_fwd_us"]
        except Exception as e:  # torchvision CUDA op missing: not fatal
            res["tv_err"] = str(e)[:120]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case")
    ap.add_argument("--all", action="store_true")
    ap.add_argument("--filter", default="")
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "dev_dcn.jsonl"))
    a = ap.parse_args()
    if a.case:
        print("RESULT " + json.dumps(run_case(a.case)))
        return
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "a") as f:
        for c in CASES:
            if a.filter and a.filter not in c[0]:
                continue
            t0 = time.time()
            try:
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--case", c[0]], capture_output=True, text=True,
                                   timeout=240)
                lines = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")]
                rec = json.loads(lines[-1][7:]) if lines else {"case": c[0], "rc": r.returncode, "stderr": r.stderr[-600:]}
            except subprocess.TimeoutExpired:
                rec = {"case": c[0], "timeout": True}
            rec["wall_s"] = round(time.time() - t0, 1)
            f.write(json.dumps(rec) + "\n")
            f.flush()
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
