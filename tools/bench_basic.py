"""ResNet18 / ResNet34 (BasicBlock) trunks on the GPU: eval embeddings/s at 256 x 256x128 in CUDA-graph mode next to
torch's cuDNN fp16 channels-last forward of the same weights (also graph-replayed), the training trunk's step time at
16 x 16 crops of 256x128, and layer1's conv2 (64 -> 64, 3x3, the halo-slab kernel) with and without its identity
residual.  Every time is the median of --reps windows of --iters launches, with the windows' min and max beside it.
Prints one JSON line per model with the card's name and power limit, then one line for the convolution.

    python tools/bench_basic.py [--iters 50] [--reps 5] [--conv-only]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import ctl_b200  # noqa: E402,F401
from ctl_b200 import _native as N  # noqa: E402
from ctl_b200.modelling.backbones.engine import GraphedForward, TrunkEngine  # noqa: E402
from ctl_b200.modelling.backbones.engine_train import TrunkTrainer  # noqa: E402
from oracle import basic_oracle as B  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(",")]
    except Exception:  # noqa: BLE001 - no nvidia-smi: the device name alone
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def gflop_per_image(layers, hw=(256, 128), last_stride=1):
    """Multiply-adds x 2 of every convolution, from the shapes (stem 7x7, BasicBlock 3x3 pairs, 1x1 downsamples)."""
    h, w = (hw[0] + 6 - 7) // 2 + 1, (hw[1] + 6 - 7) // 2 + 1
    f = 2 * h * w * 64 * 3 * 49
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    for _, planes, inplanes, stride, has_down in B._blocks(layers, last_stride):
        ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
        f += 2 * ho * wo * planes * (inplanes * 9 + planes * 9 + (inplanes if has_down else 0))
        h, w = ho, wo
    return f / 1e9


def time_ms(fn, iters, reps):
    """(median, min, max) over `reps` windows of the per-call time of `iters` back-to-back calls (CUDA events)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / iters)
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def spread(t):
    return [round(t[1], 4), round(t[2], 4)]


def graphed(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def layer1_conv2(iters, reps):
    """layer1 conv2 of ResNet18/34 at 256 x 64x32: 3x3 64 -> 64 + identity residual + ReLU, as the trunk runs it, and
    the same convolution without the residual.  ctl_conv2d_nhwc_f16 sends both to the halo-slab kernel."""
    L = N.lib()
    n, h, w = 256, 64, 32
    x = torch.randn(n, h, w, 64, device="cuda").half()
    r = torch.randn(n, h, w, 64, device="cuda").half()
    wt = (torch.randn(64, 3, 3, 64, device="cuda") / 24).half()
    b = torch.zeros(64, device="cuda")
    out = torch.empty_like(x)

    def run(res):
        N.check(L.ctl_conv2d_nhwc_f16(x.data_ptr(), n, h, w, 64, wt.data_ptr(), b.data_ptr(), N.ptr(res), out.data_ptr(),
                                      64, 3, 1, 1, 0, N.stream_ptr()))

    with_res = time_ms(lambda: run(r), iters, reps)
    no_res = time_ms(lambda: run(None), iters, reps)
    return {"layer1_conv2_residual_ms": round(with_res[0], 4), "layer1_conv2_residual_min_max": spread(with_res),
            "layer1_conv2_no_residual_ms": round(no_res[0], 4), "layer1_conv2_no_residual_min_max": spread(no_res),
            "layer1_conv2_gflop": round(2 * n * h * w * 64 * 64 * 9 / 1e9, 2), "iters": iters, "reps": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--conv-only", action="store_true", help="only the layer1 conv2 line (2000 launches per window)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_basic.py needs a GPU"
    name, power = card()
    torch.backends.cudnn.benchmark = True
    conv_line = {"gpu": name, "power_limit": power}
    conv_line.update(layer1_conv2(max(2000, args.iters), args.reps))
    if args.conv_only:
        print(json.dumps(conv_line), flush=True)
        return
    for mname, layers in B.BASIC_LAYERS.items():
        sd = B.make_trunk_state(seed=0, layers=layers)
        bs = 256
        x = torch.randn(bs, 3, 256, 128, device="cuda")
        eng = TrunkEngine(sd, "cuda", layers=layers, block="basic")
        gf = GraphedForward(eng, x, want_emb=False)
        ms_t = time_ms(gf, args.iters, args.reps)
        ms = ms_t[0]
        # torch / cuDNN: the same eval trunk (BatchNorm unfolded, as model.half().eval() runs it) in fp16 channels-last
        sdh = {k: (v.cuda().half().contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v.cuda().half())
               for k, v in sd.items() if v.is_floating_point()}
        xh = x.half().contiguous(memory_format=torch.channels_last)

        def torch_fwd():
            with torch.no_grad():
                return B.trunk_forward(xh, sdh, layers=layers).mean(dim=(2, 3))

        ref = torch_fwd().float()
        ours = gf()["global_feat"]
        torch_t = time_ms(graphed(torch_fwd), args.iters, args.reps)
        torch_ms = torch_t[0]
        # training trunk: forward + backward of 16 x 16 crops at 256x128 (graph replay)
        params = {k: v.clone().cuda() for k, v in sd.items() if v.is_floating_point()}
        tr = TrunkTrainer("cuda", layers=layers, graphs=True, block="basic")
        df = torch.randn(256, 512, device="cuda") * 1e-3

        def step():
            tr.forward(x, params)
            tr.backward(df)

        train_t = time_ms(step, max(5, args.iters // 5), args.reps)
        gfl = gflop_per_image(layers)
        line = {"gpu": name, "power_limit": power, "model": mname, "batch": bs, "hw": [256, 128],
                "gflop_per_img": round(gfl, 3),
                "eval_graph_ms": round(ms, 3), "eval_graph_min_max": spread(ms_t), "eval_emb_per_s": round(bs / ms * 1e3),
                "eval_tflops": round(bs * gfl / ms, 1),
                "torch_cudnn_fp16_cl_graph_ms": round(torch_ms, 3), "torch_cudnn_min_max": spread(torch_t),
                "torch_cudnn_emb_per_s": round(bs / torch_ms * 1e3),
                "speedup_vs_cudnn": round(torch_ms / ms, 2),
                "feat_rel_diff_vs_cudnn": float((ours - ref).abs().max() / ref.abs().max()),
                "train_step_ms_16x16": round(train_t[0], 2), "train_step_min_max": spread(train_t)}
        print(json.dumps(line), flush=True)
    print(json.dumps(conv_line), flush=True)


if __name__ == "__main__":
    main()
