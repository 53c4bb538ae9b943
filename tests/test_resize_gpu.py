"""GPU: `T.Resize` on the device (ctl_resize_bilinear_u8 through datasets/transforms.resize_batch) against Pillow's
BILINEAR `Image.resize`, bit for bit, per image and as ragged batches; mock rows, entries outside the buffer, CUDA-graph
replay; and the resized batch through forward_u8, augment_batch and run_inference at the bench shapes."""
import numpy as np
import pytest
import torch

from oracle import ctl_oracle as O
from test_modules_gpu import _Cfg, _cfg
from test_resize_cpu import KINDS, TARGETS, duke_sizes, make_image, pil_resize, sweep_sources

pytestmark = pytest.mark.gpu


def _T():
    from ctl_b200.datasets import transforms as T

    return T


def _device_resize(images, size):
    T = _T()
    return T.resize_batch(T.pack_images(images, pin=False).to("cuda"), size).cpu().numpy()


@pytest.mark.parametrize("target", TARGETS, ids=lambda t: "identity" if t is None else f"{t[0]}x{t[1]}")
def test_matches_pil_per_image_and_in_one_ragged_call(target):
    batch, refs = [np.zeros((1, 1, 3), np.uint8) + 7], []  # a 3-byte first image: every later offset is unaligned
    for h, w in sweep_sources():
        oh, ow = (h, w) if target is None else target
        for kind in KINDS:
            img = make_image(kind, h, w)
            ref = pil_resize(img, oh, ow)
            got = _device_resize([img], (oh, ow))[0]
            assert np.array_equal(got, ref), (h, w, oh, ow, kind)
            batch.append(img)
            refs.append(ref)
        batch.append(None)  # a mock row after every source
        refs.append(None)
    if target is None:
        return  # one output size per call
    T = _T()
    packed = T.pack_images(batch, pin=False)
    offs = packed.table[:, 0].numpy()
    assert (offs[1:][packed.table[1:, 1].numpy() > 0] % 2 == 1).any()
    out = T.resize_batch(packed.to("cuda"), target).cpu().numpy()
    assert np.array_equal(out[0], pil_resize(batch[0], *target))
    for i, ref in enumerate(refs):
        if ref is None:
            assert not out[i + 1].any()
        else:
            assert np.array_equal(out[i + 1], ref), (i, batch[i + 1].shape, target)


def test_batch_invariance_duke_like_256():
    sizes = duke_sizes(256, seed=11)
    imgs = [make_image("random", h, w, seed=i) for i, (h, w) in enumerate(sizes)]
    whole = _device_resize(imgs, (256, 128))
    for i, img in enumerate(imgs):
        alone = _device_resize([img], (256, 128))[0]
        assert np.array_equal(whole[i], alone), (i, img.shape)
        if i % 16 == 0:
            assert np.array_equal(alone, pil_resize(img, 256, 128)), (i, img.shape)


def test_entry_outside_the_buffer_gives_zeros_status_and_value_error():
    T = _T()
    imgs = [make_image("random", h, w, seed=i) for i, (h, w) in enumerate(duke_sizes(6, seed=3))]
    r = T.pack_images(imgs, pin=False).to("cuda")
    r.table[2, 0] = r.data.numel() - 10  # its extent runs past the end of the buffer
    with pytest.raises(ValueError, match="outside"):
        T.resize_batch(r, (256, 128))
    out = torch.full((6, 256, 128, 3), 99, dtype=torch.uint8, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(T.resize_workspace_bytes(r, (256, 128)), dtype=torch.uint8, device="cuda")
    T._resize_enqueue(r, out, status, ws)
    assert int(status.item()) == 1
    got = out.cpu().numpy()
    assert not got[2].any()
    for i in (0, 1, 3, 4, 5):
        assert np.array_equal(got[i], pil_resize(imgs[i], 256, 128)), i
    # a workspace too short for the later images: those are zeros and bit 1 is set, the ones that fit stay exact
    r = T.pack_images(imgs, pin=False).to("cuda")
    rows_fit = imgs[0].shape[0] + imgs[1].shape[0]
    ws = torch.empty(rows_fit * 128 * 3, dtype=torch.uint8, device="cuda")
    T._resize_enqueue(r, out, status, ws)
    assert int(status.item()) == 2
    got = out.cpu().numpy()
    assert np.array_equal(got[0], pil_resize(imgs[0], 256, 128)) and np.array_equal(got[1], pil_resize(imgs[1], 256, 128))
    assert not got[2:].any()


def test_graph_replay_equals_eager():
    T = _T()
    imgs = [make_image("random", h, w, seed=i) for i, (h, w) in enumerate(duke_sizes(64, seed=5))]
    imgs[7] = None
    r = T.pack_images(imgs, pin=False).to("cuda")
    eager = T.resize_batch(r, (320, 320))
    out = torch.empty_like(eager)
    status = torch.ones(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(T.resize_workspace_bytes(r, (320, 320)), dtype=torch.uint8, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        T._resize_enqueue(r, out, status, ws)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        T._resize_enqueue(r, out, status, ws)
    out.zero_()
    status.fill_(5)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager) and int(status.item()) == 0


def _pil_crops(imgs, size):
    return torch.from_numpy(np.stack([pil_resize(im, *size) for im in imgs]))


@pytest.mark.parametrize("ibn,n,size", [(False, 256, (256, 128)), (True, 128, (320, 320))], ids=["r50", "ibn-a"])
def test_forward_u8_of_device_resize_equals_pil_crops(ibn, n, size):
    from ctl_b200.modelling.backbones.engine import TrunkEngine

    T = _T()
    if ibn:
        imgs = [make_image("random", h, w, seed=i) for i, (h, w) in enumerate(duke_sizes(n, seed=21))]
    else:
        imgs = [make_image("random", 128, 64, seed=i) for i in range(n)]
    resized = T.resize_batch(T.pack_images(imgs).to("cuda"), size)
    crops = _pil_crops(imgs, size).cuda()
    assert torch.equal(resized, crops)
    eng = TrunkEngine(O.make_trunk_state(seed=2, ibn=ibn), "cuda", ibn=ibn)
    a = eng.forward_u8(resized)["global_feat"]
    b = eng.forward_u8(crops)["global_feat"]
    assert torch.equal(a, b)


def test_augment_of_device_resize_equals_augment_of_pil_crops():
    T = _T()
    imgs = [make_image("random", h, w, seed=i) for i, (h, w) in enumerate(duke_sizes(48, seed=8))]
    imgs[5] = None
    params = T.sample_params(48, 256, 128, is_real=[0 if im is None else 1 for im in imgs], rng=np.random.default_rng(2))
    resized = T.resize_batch(T.pack_images(imgs).to("cuda"), (256, 128))
    crops = torch.stack([torch.zeros(256, 128, 3, dtype=torch.uint8) if im is None
                         else torch.from_numpy(pil_resize(im, 256, 128)) for im in imgs]).cuda()
    assert torch.equal(resized, crops)
    assert torch.equal(T.augment_batch(resized, params), T.augment_batch(crops, params))


def test_run_inference_over_ragged_images_equals_pil_crops():
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
    imgs = [make_image("random", h, w, seed=i) for i, (h, w) in enumerate(duke_sizes(12, seed=9))]
    paths = [f"/data/{i:04d}_c1.jpg" for i in range(12)]
    chunks = [(i, min(i + 5, 12)) for i in range(0, 12, 5)]
    ragged = [(T.pack_images(imgs[a:b]), [""] * (b - a), paths[a:b]) for a, b in chunks]
    floats = [(T.normalize_batch(_pil_crops(imgs[a:b], (256, 128)).cuda()), [""] * (b - a), paths[a:b]) for a, b in chunks]
    emb_r, p_r = IU.run_inference(model, ragged, cfg, print_freq=10)
    emb_f, p_f = IU.run_inference(model, floats, cfg, print_freq=10)
    assert emb_r.shape == (12, 2048) and list(p_r) == list(p_f) == paths
    assert np.array_equal(emb_r, emb_f)
    feat_r, _ = IU._inference(model, ragged[0], normalize_with_bn=False, cfg=cfg)
    feat_f, _ = IU._inference(model, floats[0], normalize_with_bn=False)
    assert torch.equal(feat_r, feat_f)
    with pytest.raises(ValueError):
        IU._inference(model, ragged[0])  # a ragged batch needs the cfg's size and normalisation
