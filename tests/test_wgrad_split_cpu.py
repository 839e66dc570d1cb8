"""Host-only: which layers b2c_conv_backward_filter_split pre-splits (b2c_debug_wgrad_plan out[6]) and the split buffer size
b2c_conv_wgrad_split_bytes asks for: hi and lo bf16 planes of dY, [N][O][HWp] each, with the pixel pitch HWp padded to whole
64-pixel K blocks (7x7 maps included)."""
import ctypes as C

import caffe_mpi_b200 as m
from caffe_mpi_b200 import capi


def desc(N, Cin, H, O, k, s=1):
    return m.ConvDesc(m.ConvParams.make(N, Cin, H, H, O, k, s, k // 2, 1, 1, False))


def test_split_bytes_pad_each_image_to_whole_k_blocks():
    for N, Cin, H, O in ((64, 64, 56, 64), (64, 256, 14, 256), (64, 512, 7, 512), (3, 84, 10, 200)):
        d = desc(N, Cin, H, O, 3)
        hwp = -(-H * H // 64) * 64
        assert d.wgrad_plan()["presplit_dy"]
        assert d.wgrad_split_bytes() == 2 * 2 * N * O * hwp


def test_presplit_only_for_3x3_with_eight_or_more_channel_tiles():
    assert desc(8, 57, 16, 64, 3).wgrad_plan()["presplit_dy"]            # 8 channel tiles of 8
    assert not desc(8, 56, 16, 64, 3).wgrad_plan()["presplit_dy"]        # 7
    assert desc(8, 56, 16, 64, 3).wgrad_split_bytes() == 0
    for k, s in ((1, 1), (1, 2)):                                         # staged and compacted 1x1 routes: never
        d = desc(8, 2048, 14, 2048, k, s)
        assert not d.wgrad_plan()["presplit_dy"] and d.wgrad_split_bytes() == 0
    d = m.ConvDesc(m.ConvParams.make(8, 64, 16, 16, 64, 3, 1, 1, 1, 1, False), capi.ENGINE_CAFFE)
    assert d.wgrad_split_bytes() == 0


def test_plan_field_seven_is_optional():
    d = desc(8, 64, 16, 64, 3)
    six, seven = (C.c_int * 6)(), (C.c_int * 7)(*([-5] * 7))
    assert m.lib().b2c_debug_wgrad_plan(d._h, six, 6) == 0
    assert m.lib().b2c_debug_wgrad_plan(d._h, seven, 7) == 0
    assert list(six) == list(seven)[:6] and seven[6] == 1
