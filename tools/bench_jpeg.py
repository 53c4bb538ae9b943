"""JPEG decode on the device (datasets/transforms.decode_batch, ctl_jpeg_decode) at B = 256, and what it does to the
eval pipeline.  Sources are seeded smooth colour fields (photograph-like spectra) saved by Pillow at quality 90, 4:2:0.

  decode : the decode call alone (three launches, replayed from a CUDA graph) for Market-like 128x64 crops, a Duke-like
           ragged batch of seeded sizes between 60x30 and 400x200, and ~500 px sources (seeded sizes between 400x250
           and 600x350); windows of --replays replays alternated with the ResNet50 eval step (TrunkEngine.forward_u8,
           graph) at the shape the decoded batch is resized to (256x128), so the decode's share of the step is read off
           the same windows.  With --parent-lib, the same decode by another build of libctl_b200.so (the C ABI is
           the same) runs in the same alternation, so two builds are compared in one process.
  profile: with --profile DIR (a run of its own: tracing slows the host), torch.profiler's per-kernel device time of
           the decode's three launches for each case (and for --parent-lib's), averaged over --replays calls; the
           trace is written under DIR.
  e2e    : eval end to end from pinned HOST buffers, double-buffered (H2D of step i + 1 on a copy stream overlaps step
           i; embeddings copied back on a third stream): pinned 128x64 JPEG bytes -> H2D -> decode -> resize ->
           forward_u8 -> D2H, in windows alternated with the same pipeline from pinned native-size decoded 128x64
           images (H2D -> resize -> forward_u8 -> D2H).  H2D bytes per image for both.
  host   : Pillow's Image.open(BytesIO).convert("RGB") + np.asarray per image on one host core (the work the device
           path takes off the loader), and the host's core count.
Every line is JSON with the card's name and power limit and the mean JPEG bytes per image; times are medians of
--windows windows with their range.

    python tools/bench_jpeg.py [--windows 7] [--replays 50] [--steps 20] [--parent-lib PATH] [--profile DIR]
"""
import argparse
import io
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

import ctl_b200  # noqa: E402,F401
from ctl_b200.datasets import transforms as T  # noqa: E402
from ctl_b200.modelling.backbones.engine import GraphedCall  # noqa: E402
from tools.bench_basic import card  # noqa: E402
from tools.bench_resize import engine, med, window_ms  # noqa: E402

B = 256
SIZE = (256, 128)


def smooth(h, w, seed):
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    r = 128 + 100 * np.sin(x / 9.0 + seed) * np.cos(y / 13.0)
    g = 128 + 90 * np.cos((x + y) / 17.0 + seed)
    b = 128 + 80 * np.sin(y / 7.0 - seed) * np.sin(x / 23.0)
    noise = np.random.default_rng(seed).normal(0, 6, (h, w, 3))
    return np.clip(np.stack([r, g, b], -1) + noise, 0, 255).astype(np.uint8)


def jpeg(img):
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, "JPEG", quality=90, subsampling=2)
    return buf.getvalue()


def files(case, seed):
    rng = np.random.default_rng(seed)
    if case == "market_128x64":
        sizes = [(128, 64)] * B
    elif case == "duke_ragged":
        sizes = list(zip(rng.integers(60, 401, B), rng.integers(30, 201, B)))
    else:
        sizes = list(zip(rng.integers(400, 601, B), rng.integers(250, 351, B)))
    return [jpeg(smooth(int(h), int(w), seed * 1000 + i)) for i, (h, w) in enumerate(sizes)]


class GraphedDecode:
    """decode of one device JpegBatch into static buffers, replayed from a CUDA graph; the status is checked once.
    `fn`: the ctl_jpeg_decode of another library build (default: the tree's)."""

    def __init__(self, batch, fn=None):
        self.batch = batch
        self.out = torch.empty(max(batch.out_bytes, 1), dtype=torch.uint8, device="cuda")
        self.status = torch.zeros(len(batch), dtype=torch.int32, device="cuda")
        self.ws = torch.empty(batch.workspace_bytes, dtype=torch.uint8, device="cuda")
        self.fn = fn
        self.call = GraphedCall(self.enqueue, "cuda")

    def enqueue(self):
        if self.fn is None:
            return T._decode_enqueue(self.batch, self.out, self.status, self.ws)
        b = self.batch
        rc = self.fn(b.data.data_ptr(), b.data.numel(), b.entries.data_ptr(), len(b), b.out_table.data_ptr(),
                     self.out.data_ptr(), b.out_bytes, self.status.data_ptr(), self.ws.data_ptr(), self.ws.numel(),
                     torch.cuda.current_stream().cuda_stream)
        assert rc == 0, rc

    def __call__(self):
        self.call()
        return self.out

    def check(self):
        assert not self.status.any(), "decode status set"


CASES = ("market_128x64", "duke_ragged", "about_500px")


def parent_decoder(a):
    if not a.parent_lib:
        return None
    from tools.make_jpeg_corrupt_golden import library

    return library(a.parent_lib)


def bench_decode(a, eng, name, power):
    parent = parent_decoder(a)
    for case in CASES:
        fs = files(case, 1)
        batch = T.pack_jpegs(fs).to("cuda")
        dec = GraphedDecode(batch)
        ref = T.decode_batch(batch)
        dec()
        assert torch.equal(dec.out, ref.data)
        old = None
        if parent is not None:
            old = GraphedDecode(batch, parent)
            old()
            assert torch.equal(old.out, ref.data), "the two builds decode differently"
        data, table = ref.data.cpu().numpy(), ref.table.cpu().numpy()
        for i in range(0, B, 51):  # spot check against Pillow
            o, h, w = table[i]
            pil = np.asarray(Image.open(io.BytesIO(fs[i])).convert("RGB"))
            assert np.array_equal(data[o: o + h * w * 3].reshape(h, w, 3), pil)
        crops = T.resize_batch(ref, SIZE)
        step = GraphedCall(lambda: eng.forward_u8(crops, want_emb=True), "cuda")
        t_dec, t_step, t_old = [], [], []
        for _ in range(a.windows):
            t_dec.append(window_ms(dec, a.replays))
            t_step.append(window_ms(step, max(a.replays // 10, 3)))
            if old is not None:
                t_old.append(window_ms(old, max(a.replays // 10, 3)))
        dec.check()
        ms, rng = med(t_dec)
        sms, srng = med(t_step)
        extra = {}
        if old is not None:
            old.check()
            oms, orng = med(t_old)
            extra = {"parent_decode_ms": oms, "parent_decode_ms_range": orng, "speedup": round(oms / ms, 2),
                     "parent_decode_over_step": round(oms / sms, 4)}
        print(json.dumps({"bench": "decode", "case": case, "B": B, "decode_ms": ms, "decode_ms_range": rng, **extra,
                          "decoded_pixels": int(ref.rows and (table[:, 1] * table[:, 2]).sum()),
                          "mean_jpeg_bytes": round(float(np.mean([len(f) for f in fs])), 1),
                          "eval_step_ms_forward_u8_256x128": sms, "eval_step_ms_range": srng,
                          "decode_over_step": round(ms / sms, 4), "card": name, "power_limit": power}), flush=True)


def bench_e2e(a, eng, name, power):
    fs = files("market_128x64", 7)
    host_jpeg = T.pack_jpegs(fs)  # pinned
    host_native = T.pack_images([np.asarray(Image.open(io.BytesIO(f)).convert("RGB")) for f in fs])
    d2h_stream, copy_stream = torch.cuda.Stream(), torch.cuda.Stream()

    def pipeline(kind):
        host = host_jpeg if kind == "jpeg" else host_native
        stage = [host.to("cuda") for _ in range(2)]  # same tables; the data buffers are refilled every step
        outs = [torch.empty(B, SIZE[0], SIZE[1], 3, dtype=torch.uint8, device="cuda") for _ in range(2)]
        rs_status = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(2)]
        if kind == "jpeg":
            decoded = [torch.empty(host.out_bytes, dtype=torch.uint8, device="cuda") for _ in range(2)]
            dec_status = [torch.zeros(B, dtype=torch.int32, device="cuda") for _ in range(2)]
            dec_ws = [torch.empty(host.workspace_bytes, dtype=torch.uint8, device="cuda") for _ in range(2)]
            ragged = [T.RaggedImages(decoded[b], stage[b].out_table, host.rows) for b in range(2)]
        else:
            ragged = stage
        rs_ws = [torch.empty(T.resize_workspace_bytes(r, SIZE), dtype=torch.uint8, device="cuda") for r in ragged]

        def fwd(b):
            if kind == "jpeg":
                T._decode_enqueue(stage[b], decoded[b], dec_status[b], dec_ws[b])
            T._resize_enqueue(ragged[b], outs[b], rs_status[b], rs_ws[b])
            return eng.forward_u8(outs[b], want_emb=True)

        graphs = [GraphedCall(lambda b=b: fwd(b), "cuda") for b in range(2)]
        src, dst = host.data, [s.data for s in stage]
        out_host = [torch.empty(B, 2048).pin_memory() for _ in range(2)]
        ready, done, emb_ready, d2h_done = ([torch.cuda.Event() for _ in range(2)] for _ in range(4))
        for b in range(2):
            done[b].record()
            d2h_done[b].record()

        def prefetch(i):
            b = i % 2
            with torch.cuda.stream(copy_stream):
                copy_stream.wait_event(done[b])
                dst[b].copy_(src, non_blocking=True)
                ready[b].record(copy_stream)

        def run(steps):
            cur = torch.cuda.current_stream()
            prefetch(0)
            for i in range(steps):
                b = i % 2
                if i + 1 < steps:
                    prefetch(i + 1)
                cur.wait_event(ready[b])
                cur.wait_event(d2h_done[b])
                emb = graphs[b]()["emb"]
                done[b].record()
                emb_ready[b].record()
                with torch.cuda.stream(d2h_stream):
                    d2h_stream.wait_event(emb_ready[b])
                    out_host[b].copy_(emb, non_blocking=True)
                    d2h_done[b].record(d2h_stream)
            cur.wait_stream(d2h_stream)
            torch.cuda.synchronize()

        def window():
            t0 = time.perf_counter()
            run(a.steps)
            return B * a.steps / (time.perf_counter() - t0)

        run(3)  # warm-up
        assert all(int(s.item()) == 0 for s in rs_status), "resize status set"
        if kind == "jpeg":
            assert all(not s.any() for s in dec_status), "decode status set"
        table_bytes = host.entries.numel() + host.out_table.numel() * 8 if kind == "jpeg" else host.table.numel() * 8
        keep = (stage, outs, rs_status, rs_ws, graphs, ragged) + ((decoded, dec_status, dec_ws) if kind == "jpeg" else ())
        return window, src.numel() + table_bytes, keep

    win_j, bytes_j, keep_j = pipeline("jpeg")
    win_n, bytes_n, keep_n = pipeline("native")
    r_j, r_n = [], []
    for _ in range(a.windows):
        r_j.append(win_j())
        r_n.append(win_n())
    mean_jpeg = round(float(np.mean([len(f) for f in fs])), 1)
    for label, r, nb in (("jpeg_128x64_decoded_on_device", r_j, bytes_j), ("native_128x64_decoded_on_host", r_n, bytes_n)):
        v, rng = med(r)
        print(json.dumps({"bench": "e2e", "input": label, "B": B, "steps_per_window": a.steps, "out": list(SIZE),
                          "emb_per_s": round(v, 1), "emb_per_s_range": [round(x, 1) for x in rng],
                          "h2d_bytes_per_image": round(nb / B, 1), "mean_jpeg_bytes": mean_jpeg, "card": name,
                          "power_limit": power}), flush=True)


def bench_host(a, name, power):
    for case in ("market_128x64", "about_500px"):
        fs = files(case, 3)[:32]
        ts = []
        for _ in range(a.windows):
            t0 = time.perf_counter()
            for f in fs:
                with Image.open(io.BytesIO(f)) as im:
                    np.asarray(im.convert("RGB"))
            ts.append((time.perf_counter() - t0) / len(fs) * 1e3)
        ms, rng = med(ts)
        print(json.dumps({"bench": "host_pillow_decode", "case": case, "ms_per_image_one_core": ms, "ms_range": rng,
                          "mean_jpeg_bytes": round(float(np.mean([len(f) for f in fs])), 1),
                          "host_cores": os.cpu_count(), "usable_cores": len(os.sched_getaffinity(0)), "card": name,
                          "power_limit": power}), flush=True)


def profile_decode(a, name, power):
    """per-kernel device time of the decode's launches, from torch.profiler, for each case and build"""
    from torch.profiler import ProfilerActivity, profile

    parent = parent_decoder(a)
    os.makedirs(a.profile, exist_ok=True)
    for case in CASES:
        batch = T.pack_jpegs(files(case, 1)).to("cuda")
        for build, fn in (("this", None), ("parent", parent)):
            if build == "parent" and fn is None:
                continue
            dec = GraphedDecode(batch, fn)
            n = a.replays if build == "this" else max(a.replays // 10, 3)
            for _ in range(3):
                dec.enqueue()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(n):
                    dec.enqueue()
                torch.cuda.synchronize()
            prof.export_chrome_trace(os.path.join(a.profile, f"jpeg_{case}_{build}.pt.trace.json"))
            per = {}
            for ev in prof.key_averages():
                if "jpeg" in ev.key:
                    t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                    per[ev.key.split("(")[0].split("::")[-1]] = round(t / n / 1e3, 4)
            print(json.dumps({"bench": "decode_profile", "case": case, "build": build, "B": B, "calls": n,
                              "ms_per_call": per, "card": name, "power_limit": power}), flush=True)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--windows", type=int, default=7)
    p.add_argument("--replays", type=int, default=50)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--parent-lib", default=None, help="another build of libctl_b200.so to time beside this one")
    p.add_argument("--profile", default=None, help="directory for a torch.profiler run of the decode (only that)")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_jpeg.py needs a CUDA device")
    name, power = card()
    if a.profile:
        profile_decode(a, name, power)
        return
    eng = engine()
    bench_decode(a, eng, name, power)
    bench_e2e(a, eng, name, power)
    bench_host(a, name, power)


if __name__ == "__main__":
    main()
