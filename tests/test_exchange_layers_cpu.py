"""Size of the peer-exchange block with layers (vpt_comm_p2p_block_bytes, pure host code): the header, the accumulators, the optional
display words, the adaptive planes and tile counts, then one 256-byte-aligned full-frame plane per exported layer in VPT_LAYER_* bit order
(4 B per pixel for depth and alpha, 12 B for the volume AOV and the four light groups)."""
import ctypes as C
import itertools

import pytest

import vpt_b200 as V

LAYERS = V._native.LAYER_BITS


def rnd(b):
    return (b + 255) // 256 * 256


def base_bytes(w, h, display):
    """The block vpt_comm_p2p_export allocates: 512-byte header | float3 accum | u32 display (with display) | u32 pass counts | f32
    errors | 16 u32 tile counts, each part on a 256-byte boundary."""
    px = w * h
    return 512 + rnd(12 * px) + (rnd(4 * px) if display else 0) + 2 * rnd(4 * px) + 4 * 16


def layout_bytes(w, h, display, mask):
    end = base_bytes(w, h, display)
    if mask == 0:
        return end
    end = rnd(end)
    for name, bit in LAYERS.items():
        if mask & bit:
            end += rnd((4 if name in ("depth", "alpha") else 12) * w * h)
    return end


def block_bytes(w, h, display, mask):
    out = C.c_size_t(0)
    rc = V.lib.vpt_comm_p2p_block_bytes(w, h, display, mask, C.byref(out))
    assert rc == 0, V.lib.vpt_last_error(None)
    return out.value


SIZES = [(1, 1), (333, 197), (17, 3), (1920, 1080), (4095, 2049), (65535, 7)]


def test_layer_bits_are_the_header_constants():
    assert list(LAYERS.values()) == [1 << k for k in range(7)]
    assert list(LAYERS)[3:] == list(V.LIGHT_GROUPS)


@pytest.mark.parametrize("w,h", SIZES)
def test_block_bytes_is_the_layout_sum_for_every_mask(w, h):
    for display, mask in itertools.product((0, 1), range(128)):
        assert block_bytes(w, h, display, mask) == layout_bytes(w, h, display, mask), (w, h, display, hex(mask))


@pytest.mark.parametrize("w,h", SIZES)
def test_no_layers_is_the_block_of_vpt_comm_p2p_export(w, h):
    for display in (0, 1):
        assert block_bytes(w, h, display, 0) == base_bytes(w, h, display)


def test_all_layers_add_68_bytes_per_pixel():
    w, h = 1920, 1080
    extra = block_bytes(w, h, 1, 0x7F) - block_bytes(w, h, 1, 0)
    assert 68 * w * h <= extra < 68 * w * h + 8 * 256
    print(f"1920x1080: {extra / 1e6:.1f} MB of layers per block")


def test_refusals():
    out = C.c_size_t(0)
    assert V.lib.vpt_comm_p2p_block_bytes(64, 64, 1, 0x80, C.byref(out)) == -1
    assert b"unknown layer" in V.lib.vpt_last_error(None)
    assert V.lib.vpt_comm_p2p_block_bytes(64, 64, 1, 0xFFFFFFFF, C.byref(out)) == -1
    assert V.lib.vpt_comm_p2p_block_bytes(0, 64, 1, 1, C.byref(out)) == -1
    assert V.lib.vpt_comm_p2p_block_bytes(64, 64, 1, 1, None) == -1
