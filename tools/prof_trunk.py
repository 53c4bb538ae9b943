"""Per-launch profile of the eval trunk (last_stride 1, BN head), by default ResNet50 at the bench shape (bs 256, 256x128).

--ibn profiles ResNet50-IBN-a and --size sets the crop, e.g. --ibn --size 320x320 --batch 128 (config 4's per-GPU eval
shape).

Runs eager forwards under torch.profiler (CUDA activities only) and lists every kernel of one forward in walk order:
layer/block/role, M, K, Cout, n-tiles, the time the launch adds to the forward, its FLOPs, its algorithmic bytes (each
input read once, the output written once, plus the residual, the weights and a chained launch's second output) and the
larger of the two bounds at the H100 SXM data-sheet peaks (989 TFLOP/s dense FP16, 3.35 TB/s HBM3).

"time" is the step from the previous kernel's end to this kernel's end, the median over the profiled forwards: with
programmatic dependent launch a kernel's prologue overlaps its predecessor's tail, so raw durations overlap and do not
add up to the forward; these steps do.  "dur" is the kernel's own duration.  The launches that are not convolutions
(stem, pools, IBN-a's InstanceNorm, head) are listed by kernel name and summed per kernel at the end.

    python tools/prof_trunk.py [--batch 256] [--ibn] [--size 256x128] [--iters 20] [--json FILE]
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

PEAK_FLOPS = 989e12  # H100 SXM, dense FP16 / BF16 tensor core
PEAK_BW = 3.35e12    # H100 SXM HBM3
LAYERS, WIDTHS = (3, 4, 6, 3), (64, 128, 256, 512)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(",")]
    except Exception:  # noqa: BLE001 - no nvidia-smi: the device name alone
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def _bn(cout, chained):
    if chained:
        return 128
    return 256 if cout % 256 == 0 else (128 if cout % 128 == 0 else 64)


def conv_walk(n, H, W, last_stride=1):
    """The convolution launches of csrc/trunk.cu run_blocks for the bottleneck ResNet50, in launch order (IBN-a runs
    the same convolutions; its InstanceNorm launches are not convolutions)."""
    h, w = H // 4, W // 4  # stem 7x7/2 + maxpool 3x3/2 on even sides
    cin = 64
    out = []

    def add(name, kernel, m, k, cout, src_bytes, res=False, chain_to=0):
        bn = 64 if kernel == "c64" else _bn(cout, chain_to > 0)
        flops = 2 * m * k * cout + 2 * m * cout * chain_to
        byts = src_bytes + 2 * k * cout + 2 * m * cout * (2 if res else 1) + 2 * m * chain_to + 2 * cout * chain_to
        out.append(dict(launch=name, kernel=kernel, M=m, K=k, Cout=cout, n_tiles=cout // bn, chain_to=chain_to,
                        flops=flops, bytes=byts))

    blocks = []
    for li, (nb, width) in enumerate(zip(LAYERS, WIDTHS)):
        stride = (1, 2, 2, last_stride)[li]
        for bi in range(nb):
            blocks.append((f"layer{li + 1}.{bi}", width, stride if bi == 0 else 1, bi == 0))
    o1_ready = False
    for i, (name, width, s, has_down) in enumerate(blocks):
        cout = 4 * width
        m1 = n * h * w
        h2, w2 = (h - 1) // s + 1, (w - 1) // s + 1
        m2 = n * h2 * w2
        if not o1_ready:
            add(f"{name}.conv1", "gemm", m1, cin, width, 2 * m1 * cin)
        add(f"{name}.conv2", "c64" if width == 64 and s == 1 else "gemm", m2, 9 * width, width, 2 * m1 * width)
        nx = blocks[i + 1][1] if i + 1 < len(blocks) else 0
        chain = nx > 0 and cout % 128 == 0 and cout <= 512 and nx in (64, 128)
        role = "conv3+downsample" if has_down else "conv3"
        srcs = 2 * m2 * width + (2 * m2 * cin if has_down else 0)  # the strided shortcut reads one pixel in s*s
        k3 = width + (cin if has_down else 0)
        if chain:
            add(f"{name}.{role}+{blocks[i + 1][0]}.conv1", "chain", m2, k3, cout, srcs, res=not has_down, chain_to=nx)
        else:
            add(f"{name}.{role}", "gemm", m2, k3, cout, srcs, res=not has_down)
        o1_ready = chain
        cin, h, w = cout, h2, w2
    return out


def kernel_kind(name):
    m = re.search(r"conv_gemm_kernel<(\d+), ?(\d+)>", name)
    if m:
        return "gemm" if m.group(2) == "0" else "chain"
    if "conv3x3_c64_kernel" in name:
        return "c64"
    return "other"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--ibn", action="store_true", help="ResNet50-IBN-a instead of ResNet50")
    ap.add_argument("--size", default="256x128", help="HxW of the input crops")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()

    import ctl_b200  # noqa: F401
    from ctl_b200 import synth
    from ctl_b200.modelling.backbones.engine import TrunkEngine
    from torch.profiler import ProfilerActivity, profile

    H, W = (int(v) for v in args.size.split("x"))
    model = "ResNet50-IBN-a" if args.ibn else "ResNet50"
    dev = torch.device("cuda", 0)
    eng = TrunkEngine(synth.make_trunk_state(seed=0, ibn=args.ibn), dev, ibn=args.ibn, last_stride=1,
                      bn_head=synth.make_head_bn(0))
    x = torch.randn(args.batch, 3, H, W, generator=torch.Generator().manual_seed(1234)).to(dev)
    for _ in range(5):
        eng.forward(x, want_emb=True)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            eng.forward(x, want_emb=True)
        torch.cuda.synchronize()
    kern = sorted(((e.time_range.start, e.time_range.end, e.name) for e in prof.events()
                   if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda t: t[0])
    per = len(kern) // args.iters
    if per * args.iters != len(kern):
        raise RuntimeError(f"{len(kern)} kernels over {args.iters} forwards")
    walk = conv_walk(args.batch, H, W)
    convs = [i for i in range(per) if kernel_kind(kern[i][2]) != "other"]
    if [kernel_kind(kern[i][2]) for i in convs] != [c["kernel"] for c in walk]:
        raise RuntimeError("profiled convolution kernels do not follow the expected walk")
    rows, ci = [], 0
    for i in range(per):
        steps, durs = [], []
        for it in range(args.iters):
            s, e, _ = kern[it * per + i]
            prev_end = kern[it * per + i - 1][1] if i > 0 else s
            steps.append(e - max(prev_end, s) if i == 0 else e - prev_end)
            durs.append(e - s)
        row = dict(time_us=statistics.median(steps), dur_us=statistics.median(durs))
        if kernel_kind(kern[i][2]) != "other":
            row.update(walk[ci])
            ci += 1
        else:
            row.update(launch=kern[i][2].split("(")[0].replace("void ", ""), kernel="other")
        rows.append(row)

    name, power = card()
    print(f"# {name}, power limit {power}; {model} eval forward, bs {args.batch}, {H}x{W}, last_stride 1; "
          f"median of {args.iters} eager forwards under torch.profiler")
    print(f"{'#':>3} {'launch':44} {'M':>6} {'K':>5} {'Cout':>5} {'nt':>3} {'time_us':>8} {'dur_us':>8} {'GFLOP':>7} "
          f"{'MB':>7} {'bound_us':>8} {'bnd':>4} {'TFLOP/s':>8} {'GB/s':>6} {'of_bnd':>6}")
    tot_t = tot_b = 0.0
    for i, r in enumerate(rows):
        tot_t += r["time_us"]
        if r["kernel"] == "other":
            print(f"{i:>3} {r['launch'][:44]:44} {'':>6} {'':>5} {'':>5} {'':>3} {r['time_us']:8.1f} {r['dur_us']:8.1f}")
            continue
        tf, tb = r["flops"] / PEAK_FLOPS * 1e6, r["bytes"] / PEAK_BW * 1e6
        r["bound_us"], r["bound"] = max(tf, tb), "flop" if tf >= tb else "hbm"
        tot_b += r["bound_us"]
        t = r["time_us"]
        print(f"{i:>3} {r['launch'][:44]:44} {r['M']:>6} {r['K']:>5} {r['Cout']:>5} {r['n_tiles']:>3} {t:8.1f} "
              f"{r['dur_us']:8.1f} {r['flops'] / 1e9:7.1f} {r['bytes'] / 1e6:7.1f} {r['bound_us']:8.1f} {r['bound']:>4} "
              f"{r['flops'] / t / 1e6:8.1f} {r['bytes'] / t / 1e3:6.0f} {r['bound_us'] / t:6.2f}")
    print(f"# forward {tot_t / 1e3:.3f} ms (sum of steps); convolution bounds sum {tot_b / 1e3:.3f} ms")
    others = {}
    for r in rows:
        if r["kernel"] == "other":
            k = others.setdefault(r["launch"], [0, 0.0, 0.0])
            k[0] += 1
            k[1] += r["time_us"]
            k[2] += r["dur_us"]
    for k, (cnt, t, d) in others.items():
        print(f"# {k}: {cnt} launches, time {t:.1f} us, dur {d:.1f} us")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": name, "power_limit": power, "model": model, "batch": args.batch, "size": [H, W],
                       "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
