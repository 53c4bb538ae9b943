"""CPU: the shape rule and argument checks of the chained 1x1 launch (ctl_conv1x1_chain_nhwc_f16); no device work."""
import ctypes as C

import pytest

import ctl_b200  # noqa: F401


def test_chain_rule_covers_the_layer1_and_layer2_boundaries_only():
    from ctl_b200 import _native as N

    L = N.lib()
    assert all(L.ctl_conv1x1_chain_supported(k, n) == 1 for k, n in ((256, 64), (256, 128), (512, 128)))
    # layer2 -> layer3 (N2 = 256), layer3 (K2 = 1024) and layer4 are not chained
    assert all(L.ctl_conv1x1_chain_supported(k, n) == 0 for k, n in ((512, 256), (1024, 256), (2048, 512), (320, 64)))


def test_chain_argument_errors_are_reported_without_a_gpu():
    from ctl_b200 import _native as N

    L = N.lib()
    one = C.c_void_p(16)
    cases = [
        lambda: L.ctl_conv1x1_chain_nhwc_f16(one, 64, None, 8, 8, 0, 1, 1, one, one, None, one, 1024, one, one, 256, 0,
                                             one, None),                                          # not chainable
        lambda: L.ctl_conv1x1_chain_nhwc_f16(one, 64, one, 8, 8, 64, 1, 1, one, one, one, one, 256, one, one, 64, 0,
                                             one, None),                                          # x2 with a residual
        lambda: L.ctl_conv1x1_chain_nhwc_f16(one, 64, one, 7, 8, 64, 2, 1, one, one, None, one, 256, one, one, 64, 0,
                                             one, None),                                          # odd H2, stride 2
        lambda: L.ctl_conv1x1_chain_nhwc_f16(one, 64, None, 8, 8, 0, 2, 1, one, one, None, one, 256, one, one, 64, 0,
                                             one, None),                                          # stride without x2
        lambda: L.ctl_conv1x1_chain_nhwc_f16(one, 48, None, 8, 8, 0, 1, 1, one, one, None, one, 256, one, one, 64, 0,
                                             one, None),                                          # Cin % 64
        lambda: L.ctl_conv1x1_chain_nhwc_f16(one, 64, None, 8, 8, 0, 1, 1, one, one, None, one, 256, one, one, 64, 16,
                                             one, None),                                          # relu_from2 % 32
        lambda: L.ctl_conv1x1_chain_nhwc_f16(one, 64, None, 8, 8, 0, 1, 1, one, one, None, one, 256, None, one, 64, 0,
                                             one, None),                                          # no W2
    ]
    for i, call in enumerate(cases):
        rc = call()
        assert rc == -1, (i, rc, L.ctl_last_error())
        with pytest.raises(ValueError):
            N.check(rc)
