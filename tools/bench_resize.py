"""`T.Resize` on the device (datasets/transforms.resize_batch, ctl_resize_bilinear_u8) at B = 256, and what it does to
the eval pipeline.

  resize  : the resize call alone (both passes, replayed from a CUDA graph) for 128x64 -> 256x128 (Market, the R50
            configs), 128x64 -> 320x320 (config 4, IBN-a) and a Duke-like ragged batch of seeded sizes between 60x30
            and 400x200 -> 256x128; windows of --replays replays alternated with the ResNet50 eval step on the
            resized batch (TrunkEngine.forward_u8, graph), so the resize's share of the step is read off the same
            windows.  Bytes: native source read, intermediate written and read, output written.
  e2e     : eval end to end from pinned HOST buffers, double-buffered like bench.py's `e2e` leg (H2D of step i + 1 on a
            copy stream overlaps step i; embeddings copied back on a third stream): pinned native-size 128x64 images ->
            H2D -> resize -> forward_u8 -> D2H, in windows alternated with the same pipeline from pinned pre-resized
            256x128 crops (bench.py's leg).  H2D bytes per image for both.
  host    : PIL.Image.resize(BILINEAR) per image on one host core (the work the device path takes off the loader),
            and the host's core count.
Every line is JSON with the card's name and power limit; times are medians of --windows windows with their range.

    python tools/bench_resize.py [--windows 7] [--replays 50] [--steps 20]
"""
import argparse
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
from ctl_b200.modelling.backbones.engine import GraphedCall, TrunkEngine  # noqa: E402
from oracle import ctl_oracle as O  # noqa: E402
from tools.bench_basic import card  # noqa: E402

B = 256


def med(ts):
    ts = sorted(ts)
    return round(ts[len(ts) // 2], 4), [round(ts[0], 4), round(ts[-1], 4)]


def window_ms(fn, reps):
    """Device time of `reps` calls of fn, CUDA events, ms per call."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def duke_images(n, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (int(h), int(w), 3), dtype=np.uint8)
            for h, w in zip(rng.integers(60, 401, n), rng.integers(30, 201, n))]


def market_images(n, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (128, 64, 3), dtype=np.uint8) for _ in range(n)]


class GraphedResize:
    """resize of one device RaggedImages into static buffers, replayed from a CUDA graph; the status is checked once."""

    def __init__(self, ragged, size):
        self.ragged = ragged
        self.out = torch.empty(len(ragged), size[0], size[1], 3, dtype=torch.uint8, device="cuda")
        self.status = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.ws = torch.empty(T.resize_workspace_bytes(ragged, size), dtype=torch.uint8, device="cuda")
        self.call = GraphedCall(lambda: T._resize_enqueue(self.ragged, self.out, self.status, self.ws), "cuda")

    def __call__(self):
        self.call()
        return self.out

    def check(self):
        assert int(self.status.item()) == 0, "resize status set"


def engine():
    sd = O.make_trunk_state(seed=0)
    g = torch.Generator().manual_seed(1)
    head = dict(weight=torch.rand(2048, generator=g) + 0.5, bias=torch.randn(2048, generator=g) * 0.1,
                running_mean=torch.randn(2048, generator=g) * 0.1, running_var=torch.rand(2048, generator=g) + 0.5)
    return TrunkEngine(sd, "cuda", bn_head=head)


def bench_resize(a, eng, name, power):
    cases = [("market_256x128", market_images(B, 0), (256, 128)), ("market_320x320", market_images(B, 0), (320, 320)),
             ("duke_ragged_256x128", duke_images(B, 1), (256, 128))]
    for label, imgs, size in cases:
        ragged = T.pack_images(imgs).to("cuda")
        rs = GraphedResize(ragged, size)
        ref = T.resize_batch(ragged, size)
        rs()
        assert torch.equal(rs.out, ref)
        for i in range(0, B, 51):  # spot check against Pillow
            pil = np.asarray(Image.fromarray(imgs[i]).resize((size[1], size[0]), Image.BILINEAR))
            assert np.array_equal(ref[i].cpu().numpy(), pil)
        step = GraphedCall(lambda: eng.forward_u8(rs.out, want_emb=True), "cuda")
        t_rs, t_step = [], []
        for _ in range(a.windows):
            t_rs.append(window_ms(rs, a.replays))
            t_step.append(window_ms(step, max(a.replays // 10, 3)))
        rs.check()
        src = sum(im.nbytes for im in imgs)
        mid = ragged.rows * size[1] * 3
        out = B * size[0] * size[1] * 3
        moved = src + 2 * mid + out
        ms, rng = med(t_rs)
        sms, srng = med(t_step)
        print(json.dumps({"bench": "resize", "case": label, "B": B, "out": list(size), "resize_ms": ms,
                          "resize_ms_range": rng, "bytes": moved, "GB_per_s": round(moved / ms / 1e6, 1),
                          "eval_step_ms_forward_u8": sms, "eval_step_ms_range": srng,
                          "resize_share_of_step": round(ms / (ms + sms), 4), "card": name, "power_limit": power}),
              flush=True)


def bench_e2e(a, eng, name, power):
    size = (256, 128)
    n_rot = 3
    native = [T.pack_images(market_images(B, 10 + i)) for i in range(n_rot)]  # pinned
    crops = [T.resize_batch(r.to("cuda"), size).cpu().pin_memory() for r in native]
    d2h_stream, copy_stream = torch.cuda.Stream(), torch.cuda.Stream()

    def pipeline(kind):
        if kind == "native":
            stage = [native[0].to("cuda") for _ in range(2)]  # same table, same byte count for every batch
            outs = [torch.empty(B, size[0], size[1], 3, dtype=torch.uint8, device="cuda") for _ in range(2)]
            status = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(2)]
            ws = [torch.empty(T.resize_workspace_bytes(s, size), dtype=torch.uint8, device="cuda") for s in stage]

            def fwd(b):
                T._resize_enqueue(stage[b], outs[b], status[b], ws[b])
                return eng.forward_u8(outs[b], want_emb=True)

            graphs = [GraphedCall(lambda b=b: fwd(b), "cuda") for b in range(2)]
            src, dst = [r.data for r in native], [s.data for s in stage]
        else:
            stage = [torch.empty(B, size[0], size[1], 3, dtype=torch.uint8, device="cuda") for _ in range(2)]
            status = []
            graphs = [GraphedCall(lambda b=b: eng.forward_u8(stage[b], want_emb=True), "cuda") for b in range(2)]
            src, dst = crops, stage
        out_host = [torch.empty(B, 2048).pin_memory() for _ in range(2)]
        ready, done, emb_ready, d2h_done = ([torch.cuda.Event() for _ in range(2)] for _ in range(4))
        for b in range(2):
            done[b].record()
            d2h_done[b].record()

        def prefetch(i):
            b = i % 2
            with torch.cuda.stream(copy_stream):
                copy_stream.wait_event(done[b])
                dst[b].copy_(src[i % n_rot], non_blocking=True)
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
        assert all(int(st.item()) == 0 for st in status), "resize status set"
        # the graphs hold raw pointers to every buffer: the caller keeps them alive (a later capture empties the cache)
        keep = (stage, status, graphs) + ((outs, ws) if kind == "native" else ())
        return window, src[0].numel() * src[0].element_size() + (native[0].table.numel() * 8 if kind == "native" else 0), keep

    win_n, bytes_n, keep_n = pipeline("native")
    win_c, bytes_c, keep_c = pipeline("crops")
    r_n, r_c = [], []
    for _ in range(a.windows):
        r_n.append(win_n())
        r_c.append(win_c())
    for label, r, nb in (("native_128x64_resized_on_device", r_n, bytes_n), ("pre_resized_256x128", r_c, bytes_c)):
        v, rng = med(r)
        print(json.dumps({"bench": "e2e", "input": label, "B": B, "steps_per_window": a.steps,
                          "emb_per_s": round(v, 1), "emb_per_s_range": [round(x, 1) for x in rng],
                          "h2d_bytes_per_image": round(nb / B, 1), "card": name, "power_limit": power}), flush=True)


def bench_host(a, name, power):
    img = Image.fromarray(market_images(1, 3)[0])
    for size in ((256, 128), (320, 320)):
        ts = []
        for _ in range(a.windows):
            t0 = time.perf_counter()
            for _ in range(200):
                img.resize((size[1], size[0]), Image.BILINEAR)
            ts.append((time.perf_counter() - t0) / 200 * 1e3)
        ms, rng = med(ts)
        print(json.dumps({"bench": "host_pil_resize", "src": [128, 64], "out": list(size), "ms_per_image_one_core": ms,
                          "ms_range": rng, "host_cores": os.cpu_count(), "usable_cores": len(os.sched_getaffinity(0)),
                          "card": name, "power_limit": power}), flush=True)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--windows", type=int, default=7)
    p.add_argument("--replays", type=int, default=50)
    p.add_argument("--steps", type=int, default=20)
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_resize.py needs a CUDA device")
    name, power = card()
    eng = engine()
    bench_resize(a, eng, name, power)
    bench_e2e(a, eng, name, power)
    bench_host(a, name, power)


if __name__ == "__main__":
    main()
