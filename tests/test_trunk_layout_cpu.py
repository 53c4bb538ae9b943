"""CPU: both trunk handles are built from one ResNet layout (csrc/resnet.h).  ctl_embed_workspace_bytes and
ctl_train_workspace_bytes are host-side walks over that layout, so the blocks, every convolution's shape and stride, the
downsamples and the IBN-a splits all enter them.  The values below are pinned: a change to the network either handle
builds changes at least one of them."""
import ctypes as C

import pytest

import ctl_b200  # noqa: F401
from ctl_b200 import _native as N

NETS = {  # name -> (block, ibn, stage_blocks)
    "r50": (N.CTL_BLOCK_BOTTLENECK, 0, (3, 4, 6, 3)),
    "r50_ibn": (N.CTL_BLOCK_BOTTLENECK, 1, (3, 4, 6, 3)),
    "r101": (N.CTL_BLOCK_BOTTLENECK, 0, (3, 4, 23, 3)),
    "bottleneck_1111": (N.CTL_BLOCK_BOTTLENECK, 0, (1, 1, 1, 1)),
    "r18": (N.CTL_BLOCK_BASIC, 0, (2, 2, 2, 2)),
    "r34": (N.CTL_BLOCK_BASIC, 0, (3, 4, 6, 3)),
    "basic_1111": (N.CTL_BLOCK_BASIC, 0, (1, 1, 1, 1)),
}
SHAPES = [(16, 256, 128), (8, 320, 320), (2, 110, 62)]  # (n, H, W)
# (name, last_stride) -> [(ctl_embed_workspace_bytes, ctl_train_workspace_bytes) for each shape of SHAPES]
BYTES = {
    ("r50", 1): [(83886080, 688160768), (131072000, 1056210944), (2293760, 37196288)],
    ("r50", 2): [(83886080, 615809024), (131072000, 947879936), (2293760, 35312128)],
    ("r50_ibn", 1): [(83886080, 688295936), (131072000, 1056274432), (2293760, 37207040)],
    ("r50_ibn", 2): [(83886080, 615944192), (131072000, 947943424), (2293760, 35322880)],
    ("r101", 1): [(83886080, 902279168), (131072000, 1390653440), (2293760, 43254272)],
    ("r101", 2): [(83886080, 829927424), (131072000, 1282322432), (2293760, 41370112)],
    ("bottleneck_1111", 1): [(83886080, 398618624), (131072000, 603877376), (2293760, 29147648)],
    ("bottleneck_1111", 2): [(83886080, 364015616), (131072000, 554528768), (2293760, 17760768)],
    ("r18", 1): [(20971520, 237598720), (32768000, 360577024), (551168, 24790784)],
    ("r18", 2): [(20971520, 221608960), (32768000, 335444992), (551168, 24375040)],
    ("r34", 1): [(20971520, 296348672), (32768000, 452357120), (551168, 26426112)],
    ("r34", 2): [(20971520, 274067456), (32768000, 417394688), (551168, 25846528)],
    ("basic_1111", 1): [(20971520, 199834624), (32768000, 301579264), (551168, 23743232)],
    ("basic_1111", 2): [(20971520, 190136320), (32768000, 286277632), (551168, 23491328)],
}


@pytest.mark.parametrize("name,last_stride", sorted(BYTES))
def test_workspace_sizes_of_both_handles_are_pinned(name, last_stride):
    L = N.lib()
    block, ibn, stages = NETS[name]
    h, t = C.c_void_p(), C.c_void_p()
    assert L.ctl_trunk_create(C.byref(h), block, ibn, last_stride, (C.c_int32 * 4)(*stages)) == 0
    assert L.ctl_trainer_create(C.byref(t), block, ibn, last_stride, 0.1, (C.c_int32 * 4)(*stages)) == 0
    try:
        got = [(L.ctl_embed_workspace_bytes(h, *s), L.ctl_train_workspace_bytes(t, *s)) for s in SHAPES]
        assert got == BYTES[(name, last_stride)]
    finally:
        L.ctl_trunk_destroy(h)
        L.ctl_trainer_destroy(t)
