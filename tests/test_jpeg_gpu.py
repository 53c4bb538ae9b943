"""GPU: JPEG decode on the device (ctl_jpeg_decode through datasets/transforms.decode_batch) against Pillow's
`Image.open(...).convert("RGB")`, bit for bit, per image and as ragged batches with raw and mock entries; per-image
errors, CUDA-graph replay; and the decoded batch through resize_batch + forward_u8, augment_batch and run_inference."""
import io

import numpy as np
import pytest
import torch
from PIL import Image

from jpeg_fixtures import duke_sizes, encode, fixtures, make_image, pillow_decode
from oracle import ctl_oracle as O
from test_modules_gpu import _Cfg, _cfg

pytestmark = pytest.mark.gpu


def _T():
    from ctl_b200.datasets import transforms as T

    return T


def _images(ragged):
    """host list of the HWC arrays of a RaggedImages (None for mock rows)"""
    data, table = ragged.data.cpu().numpy(), ragged.table.cpu().numpy()
    return [None if h == 0 else data[o: o + h * w * 3].reshape(h, w, 3) for o, h, w in table]


def test_matches_pillow_per_image():
    T = _T()
    wrong = []
    for label, data in fixtures():
        got = _images(T.decode_batch(T.pack_jpegs([data], pin=False).to("cuda")))[0]
        if not np.array_equal(got, pillow_decode(data)):
            wrong.append(label)
    assert not wrong, wrong[:20]


def test_matches_pillow_in_one_ragged_batch_with_raw_and_mock_entries():
    T = _T()
    prog = encode(make_image("random", 33, 17), 2, progressive=True)
    png = io.BytesIO()
    Image.fromarray(make_image("ramp", 12, 9)).save(png, "PNG")
    items, refs = [], []
    for i, (label, data) in enumerate(fixtures()):
        items.append(data)
        refs.append(pillow_decode(data))
        if i % 7 == 0:
            items.append(None)
            refs.append(None)
        if i % 101 == 0:
            extra = prog if i % 2 else png.getvalue()
            items.append(extra)
            refs.append(pillow_decode(extra))
    batch = T.pack_jpegs(items)
    assert len(batch.fallback) >= 2
    offsets = batch.entries[:, :8].clone().view(torch.int64).flatten().tolist()
    assert any(o % 2 for o in offsets) and any(o % 4 == 3 for o in offsets)  # packed at any byte alignment
    got = _images(T.decode_batch(batch.to("cuda")))
    assert len(got) == len(refs)
    for i, (g, r) in enumerate(zip(got, refs)):
        assert (g is None) == (r is None), i
        assert r is None or np.array_equal(g, r), i


def test_batch_invariance_market_like_256():
    T = _T()
    files = [encode(make_image("smooth" if i % 3 else "random", 128, 64, i), (0, 1, 2, "L")[i % 4],
                    quality=(75, 90, 95)[i % 3]) for i in range(256)]
    together = _images(T.decode_batch(T.pack_jpegs(files).to("cuda")))
    for i in (0, 1, 2, 3, 77, 128, 254, 255):
        alone = _images(T.decode_batch(T.pack_jpegs([files[i]]).to("cuda")))[0]
        assert np.array_equal(together[i], alone), i
    for i, f in enumerate(files):
        assert np.array_equal(together[i], pillow_decode(f)), i


def test_errors_are_per_image():
    T = _T()
    files = [encode(make_image("random", 40 + i, 30 + 2 * i, i), (0, 2, "L")[i % 3]) for i in range(6)]
    sos = files[2].find(b"\xff\xda")
    files[2] = files[2][: sos + (len(files[2]) - sos) // 2]  # entropy-coded data cut in half
    batch = T.pack_jpegs(files + [None], pin=False)
    ent = batch.entries.clone()
    ent[4, :8] = torch.tensor([batch.data.numel() - 10], dtype=torch.int64).view(torch.uint8)  # outside the buffer
    batch.entries = ent
    dev = batch.to("cuda")
    out = torch.full((batch.out_bytes,), 77, dtype=torch.uint8, device="cuda")
    status = torch.full((len(batch),), -1, dtype=torch.int32, device="cuda")
    ws = torch.empty(batch.workspace_bytes, dtype=torch.uint8, device="cuda")
    T._decode_enqueue(dev, out, status, ws)
    st = status.cpu().tolist()
    assert st == [0, 0, 1, 0, 2, 0, 0], st
    got = _images(T.RaggedImages(out, dev.out_table, batch.rows))
    for i in range(6):
        if i in (2, 4):
            assert not got[i].any(), i
        else:
            assert np.array_equal(got[i], pillow_decode(files[i])), i
    with pytest.raises(ValueError, match=r"2: corrupt .* 4: entry outside"):
        T.decode_batch(dev)
    short = torch.empty(batch.workspace_bytes - 64 * 3 * 20, dtype=torch.uint8, device="cuda")
    T._decode_enqueue(dev, out, status, short)  # the last JPEG's region no longer fits
    assert status.cpu().tolist()[5] == 8


def test_graph_replay_equals_eager():
    T = _T()
    files = [encode(make_image("random", h, w, i), (0, 1, 2, "L")[i % 4], restart_marker_blocks=(0, 2)[i % 2])
             for i, (h, w) in enumerate(duke_sizes(64, seed=5))]
    files[7] = None
    b = T.pack_jpegs(files).to("cuda")
    eager = T.decode_batch(b).data
    out = torch.empty_like(eager)
    status = torch.ones(len(b), dtype=torch.int32, device="cuda")
    ws = torch.empty(b.workspace_bytes, dtype=torch.uint8, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        T._decode_enqueue(b, out, status, ws)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        T._decode_enqueue(b, out, status, ws)
    out.zero_()
    status.fill_(5)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager) and not status.any()


def _pillow_ragged(files):
    T = _T()
    return T.pack_images([None if f is None else pillow_decode(f) for f in files])


@pytest.mark.parametrize("ibn,n,size", [(False, 256, (256, 128)), (True, 128, (320, 320))], ids=["r50", "ibn-a"])
def test_forward_u8_of_device_decode_equals_pillow(ibn, n, size):
    from ctl_b200.modelling.backbones.engine import TrunkEngine

    T = _T()
    if ibn:
        files = [encode(make_image("smooth", h, w, i), (0, 1, 2)[i % 3], quality=90)
                 for i, (h, w) in enumerate(duke_sizes(n, seed=21))]
    else:
        files = [encode(make_image("smooth", 128, 64, i), 2, quality=90) for i in range(n)]
    dec = T.resize_batch(T.decode_batch(T.pack_jpegs(files).to("cuda")), size)
    ref = T.resize_batch(_pillow_ragged(files).to("cuda"), size)
    assert torch.equal(dec, ref)
    eng = TrunkEngine(O.make_trunk_state(seed=2, ibn=ibn), "cuda", ibn=ibn)
    assert torch.equal(eng.forward_u8(dec)["global_feat"], eng.forward_u8(ref)["global_feat"])


def test_augment_after_device_decode_equals_augment_after_pillow():
    T = _T()
    files = [encode(make_image("random", h, w, i), (0, 2)[i % 2]) for i, (h, w) in enumerate(duke_sizes(48, seed=8))]
    files[5] = None
    params = T.sample_params(48, 256, 128, is_real=[0 if f is None else 1 for f in files],
                             rng=np.random.default_rng(2))
    dec = T.resize_batch(T.decode_batch(T.pack_jpegs(files).to("cuda")), (256, 128))
    ref = T.resize_batch(_pillow_ragged(files).to("cuda"), (256, 128))
    assert torch.equal(T.augment_batch(dec, params), T.augment_batch(ref, params))


def test_run_inference_over_jpeg_batches_equals_ragged_images():
    from ctl_b200.inference import inference_utils as IU
    from ctl_b200.modelling.ctl_model import CTLModel

    T = _T()
    cfg = _cfg(TEST__IMS_PER_BATCH=5)
    cfg["INPUT"] = _Cfg(SIZE_TEST=[256, 128], PIXEL_MEAN=[0.485, 0.456, 0.406], PIXEL_STD=[0.229, 0.224, 0.225])
    torch.manual_seed(0)
    model = CTLModel(cfg, num_classes=16, num_query=4).cuda().eval()
    model.backbone.base.load_state_dict(O.make_trunk_state(seed=6))
    model.backbone.invalidate()
    with torch.no_grad():
        model.bn.running_mean.normal_(0, 0.1)
        model.bn.running_var.uniform_(0.5, 1.5)
    files = [encode(make_image("smooth", h, w, i), (0, 1, 2, "L")[i % 4]) for i, (h, w) in enumerate(duke_sizes(12, seed=9))]
    paths = [f"/data/{i:04d}_c1.jpg" for i in range(12)]
    chunks = [(i, min(i + 5, 12)) for i in range(0, 12, 5)]
    jpegs = [(T.pack_jpegs(files[a:b]), [""] * (b - a), paths[a:b]) for a, b in chunks]
    ragged = [(_pillow_ragged(files[a:b]), [""] * (b - a), paths[a:b]) for a, b in chunks]
    emb_j, p_j = IU.run_inference(model, jpegs, cfg, print_freq=10)
    emb_r, p_r = IU.run_inference(model, ragged, cfg, print_freq=10)
    assert emb_j.shape == (12, 2048) and list(p_j) == list(p_r) == paths
    assert np.array_equal(emb_j, emb_r)
    with pytest.raises(ValueError):
        IU._inference(model, jpegs[0])  # a JpegBatch needs the cfg's size and normalisation
