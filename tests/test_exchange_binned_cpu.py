"""Size of the peer-exchange block with binned layers (vpt_comm_p2p_block_bytes_binned, pure host code): the block of
vpt_comm_p2p_block_bytes, then the deep slices [n_slices][H][W] float4 and the mattes [n_mattes][H][W] float4, each array on a 256-byte
boundary."""
import ctypes as C
import itertools

import pytest

import vpt_b200 as V

LAYERS = V._native.LAYER_BITS
SLICES = (0, 1, 7, 32)
MATTES = (0, 1, 5, 32)
# no layers, one f32 plane, one float3 plane, a mixed mask, all seven
MASKS = (0x00, 0x01, 0x04, 0x2B, 0x7F)
SIZES = [(1, 1), (333, 197), (17, 3), (1920, 1080), (4095, 2049), (65535, 7)]


def rnd(b):
    return (b + 255) // 256 * 256


def layout_bytes(w, h, display, mask, n_slices, n_mattes):
    """512-byte header | float3 accum | u32 display (with display) | u32 pass counts | f32 errors | 16 u32 tile counts | the layer planes
    in bit order | deep slices | mattes; every part after the tile counts starts on a 256-byte boundary."""
    px = w * h
    end = 512 + rnd(12 * px) + (rnd(4 * px) if display else 0) + 2 * rnd(4 * px) + 4 * 16
    if mask == 0 and n_slices == 0 and n_mattes == 0:
        return end
    end = rnd(end)
    for name, bit in LAYERS.items():
        if mask & bit:
            end += rnd((4 if name in ("depth", "alpha") else 12) * px)
    return end + rnd(16 * n_slices * px) + rnd(16 * n_mattes * px)


def binned_bytes(w, h, display, mask, n_slices, n_mattes):
    out = C.c_size_t(0)
    rc = V.lib.vpt_comm_p2p_block_bytes_binned(w, h, display, mask, n_slices, n_mattes, C.byref(out))
    assert rc == 0, V.lib.vpt_last_error(None)
    return out.value


def block_bytes(w, h, display, mask):
    out = C.c_size_t(0)
    assert V.lib.vpt_comm_p2p_block_bytes(w, h, display, mask, C.byref(out)) == 0, V.lib.vpt_last_error(None)
    return out.value


def test_binned_constants_are_the_header_values():
    assert (V._native.VPT_BINNED_DEEP, V._native.VPT_BINNED_MATTES) == (1, 2)
    assert V._native.VPT_DEEP_MAX_SLICES == 32 and V._native.VPT_MATTE_MAX == 32


@pytest.mark.parametrize("w,h", SIZES)
def test_block_bytes_binned_is_the_layout_sum(w, h):
    for display, mask, ns, nm in itertools.product((0, 1), MASKS, SLICES, MATTES):
        assert binned_bytes(w, h, display, mask, ns, nm) == layout_bytes(w, h, display, mask, ns, nm), (w, h, display, hex(mask), ns, nm)


@pytest.mark.parametrize("w,h", SIZES)
def test_no_binned_layers_is_the_block_of_vpt_comm_p2p_block_bytes(w, h):
    for display, mask in itertools.product((0, 1), range(128)):
        assert binned_bytes(w, h, display, mask, 0, 0) == block_bytes(w, h, display, mask), (w, h, display, hex(mask))


def test_sizes_past_32_bits():
    """K x H x W x 16 passes 2^32 long before a side reaches 65535: 32 slices of a 4096 x 2160 frame are 4.5 GB."""
    w, h = 4096, 2160
    extra = binned_bytes(w, h, 1, 0, 32, 0) - binned_bytes(w, h, 1, 0, 0, 0)
    assert extra >= 32 * 16 * w * h > 2 ** 32
    both = binned_bytes(w, h, 1, 0x7F, 32, 32) - binned_bytes(w, h, 1, 0x7F, 0, 0)
    assert both == 2 * rnd(32 * 16 * w * h)


def test_refusals():
    out = C.c_size_t(0)
    for args in ((64, 64, 1, 0, 33, 0), (64, 64, 1, 0, 0, 33), (64, 64, 1, 0, 0xFFFFFFFF, 1)):
        assert V.lib.vpt_comm_p2p_block_bytes_binned(*args, C.byref(out)) == -1, args
    assert b"n_slices" in V.lib.vpt_last_error(None)
    assert V.lib.vpt_comm_p2p_block_bytes_binned(64, 64, 1, 0, 0, 33, C.byref(out)) == -1
    assert b"n_mattes" in V.lib.vpt_last_error(None)
    assert V.lib.vpt_comm_p2p_block_bytes_binned(64, 64, 1, 0x80, 1, 1, C.byref(out)) == -1
    assert b"unknown layer" in V.lib.vpt_last_error(None)
    assert V.lib.vpt_comm_p2p_block_bytes_binned(64, 64, 1, 0, 1, 1, None) == -1
    assert V.lib.vpt_comm_p2p_block_bytes_binned(0, 64, 1, 0, 1, 1, C.byref(out)) == -1
    assert V.lib.vpt_comm_p2p_block_bytes_binned(64, 0, 1, 0, 1, 1, C.byref(out)) == -1
    assert V.lib.vpt_comm_p2p_block_bytes_binned(64, 64, 1, 0, 32, 32, C.byref(out)) == 0


def test_python_refuses_counts_out_of_range():
    from vpt_b200.renderer import _binned_counts
    assert _binned_counts(0, 0) == (0, 0) and _binned_counts(32, 1) == (32, 1)
    for bad in ((33, 0), (0, 33), (-1, 0)):
        with pytest.raises(V.VptError):
            _binned_counts(*bad)
