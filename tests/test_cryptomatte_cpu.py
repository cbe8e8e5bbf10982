"""The Cryptomatte without a GPU: the library's name hash (vpt_cryptomatte_hash) against scikit-learn's MurmurHash3 and published
vectors, the id float's exponent rule, the update and rank rules of tests/cryptomatte_ref.py against closed forms, the EXR metadata and
manifest, and the ctypes bindings (include/vpt_b200.h, DESIGN.md section 8s)."""
import ctypes as C
import json
import struct

import numpy as np
import pytest
from sklearn.utils import murmurhash3_32

import vpt_b200 as V
from vpt_b200 import _native as N
from vpt_b200.renderer import Renderer, cryptomatte_id

import cryptomatte_ref as R


def lib_hash(data: bytes):
    f = C.c_float(0.0)
    h = int(V.lib.vpt_cryptomatte_hash(data, len(data), C.byref(f)))
    return h, struct.unpack("<I", bytes(f))[0]


NAMES = ["", "a", "ab", "abc", "abcd", "abcde", "cloud.0", "cumulus_17", "dragon.999", "x" * 16, "y" * 17,
         "nuage_été", "雲.3", "\U0001f325️", "Straße-à-ñ"]


@pytest.mark.parametrize("length", range(18))
def test_hash_matches_scikit_learn_at_every_tail_length(length):
    rng = np.random.default_rng(length)
    for _ in range(20):
        data = bytes(rng.integers(0, 256, length, dtype=np.uint8))
        assert lib_hash(data)[0] == murmurhash3_32(data, seed=0, positive=True)
        assert lib_hash(data)[0] == R.murmur3_32(data)


def test_hash_of_utf8_names_matches_scikit_learn():
    for name in NAMES:
        b = name.encode("utf-8")
        assert lib_hash(b)[0] == murmurhash3_32(b, seed=0, positive=True), name


def test_published_seed0_vectors():
    assert lib_hash(b"")[0] == 0
    assert lib_hash(b"hello")[0] == 0x248BFA47
    assert lib_hash(b"The quick brown fox jumps over the lazy dog")[0] == 0x2E4FF723
    # a NULL name of length 0 is the empty name
    assert int(V.lib.vpt_cryptomatte_hash(None, 0, None)) == 0


def found_names(exponent, n=2):
    out, i = [], 0
    while len(out) < n:
        name = f"probe{i}"
        if (R.murmur3_32(name.encode()) >> 23) & 0xFF == exponent:
            out.append(name)
        i += 1
    return out


@pytest.mark.parametrize("exponent", [0, 255])
def test_exponent_0_and_255_flip_bit_23(exponent):
    for name in found_names(exponent):
        h, bits = lib_hash(name.encode())
        assert (h >> 23) & 0xFF == exponent
        assert bits == h ^ (1 << 23)
        f = struct.unpack("<f", struct.pack("<I", bits))[0]
        assert np.isfinite(f) and (f == 0.0 or abs(f) >= np.finfo(np.float32).tiny)
        assert cryptomatte_id(name)[1] == "%08x" % bits == R.manifest_hex(name)


def test_other_exponents_keep_the_hash():
    for name in NAMES + [f"n{i}" for i in range(200)]:
        h, bits = lib_hash(name.encode("utf-8"))
        if (h >> 23) & 0xFF not in (0, 255):
            assert bits == h
        assert cryptomatte_id(name)[1] == R.manifest_hex(name)
        assert np.float32(cryptomatte_id(name)[0]).tobytes() == np.float32(R.id_float(name)).tobytes()


def state_of(capacity, passes, iteration=0, max_interactions=1 << 30, state=None):
    """passes: list of ids (None = a sample without collision)"""
    st = state or R.PixelState(capacity)
    depths = [0.0 if x is None else 1.0 for x in passes]
    ids = [0 if x is None else x for x in passes]
    return R.update(st, iteration, max_interactions, depths, ids)


def test_entries_fill_in_first_seen_order():
    st = state_of(4, [7, None, 3, 7, R.SPHERE, 3, 7, 0])
    assert st.n == 8 and st.overflow == 0
    assert st.ids == [7, 3, R.SPHERE, 0] and st.counts == [3, 2, 1, 1]


def test_overflow_when_full_and_existing_ids_still_count():
    st = state_of(2, [5, 6, 9, 5, 10, 6, 9])
    assert st.ids == [5, 6] and st.counts == [2, 2] and st.overflow == 3 and st.n == 7


def test_iteration_zero_clears_and_the_gate_stops():
    st = state_of(3, [1, 2, 2])
    st = state_of(3, [4, 4], iteration=0, state=st)                 # a new frame
    assert st.ids[:1] == [4] and st.counts == [2, 0, 0] and st.n == 2
    st = state_of(3, [5, 4, 5], iteration=2, max_interactions=4, state=st)   # only passes at it 2 and 3 count
    assert st.n == 4 and st.ids[:2] == [4, 5] and st.counts[:2] == [3, 1]
    before = st.words().copy()
    state_of(3, [6, 6], iteration=4, max_interactions=4, state=st)
    assert (st.words() == before).all()
    st0 = state_of(3, [1], iteration=0, max_interactions=0)          # max_interactions 0: not even the clear
    assert st0.n == 0


def test_nan_and_negative_depths_add_no_id():
    st = R.update(R.PixelState(2), 0, 100, [np.nan, -1.0, 0.0, 2.0], [9, 9, 9, 9])
    assert st.n == 4 and st.ids[0] == 9 and st.counts == [1, 0]


def test_split_calls_equal_one_call():
    rng = np.random.default_rng(3)
    passes = [None if rng.random() < 0.3 else int(rng.integers(0, 6)) for _ in range(40)]
    one = state_of(4, passes).words()
    st = R.PixelState(4)
    for a, b in ((0, 5), (5, 17), (17, 40)):
        state_of(4, passes[a:b], iteration=a, state=st)
    assert (st.words() == one).all()


def test_ranks_order_ties_by_index_sphere_last_and_empty_ranks():
    table = np.array([10.0, 11.0, 12.0, 13.0], np.float32)
    st = state_of(6, [3, 1, R.SPHERE, 1, 3, R.SPHERE, 2, 7])
    # counts: 3 -> 2, 1 -> 2, sphere -> 2, 2 -> 1, 7 (not an instance) -> 1; n = 8
    r = R.ranks(st.words(), 6, table, -5.0, 8)
    assert r.shape == (4, 4)
    assert r[0].tolist() == [11.0, 0.25, 13.0, 0.25]                 # ties by instance index
    assert r[1].tolist() == [-5.0, 0.25, 12.0, 0.125]                # the sphere last among count 2
    assert r[2].tolist() == [0.0, 0.125, 0.0, 0.0]                   # id 7 is no instance: 0.0f; then the empty rank
    assert r[3].tolist() == [0.0, 0.0, 0.0, 0.0]
    assert (R.ranks(R.PixelState(3).words(), 3, table, 1.0, 4) == 0).all()   # n == 0
    only_misses = state_of(3, [None, None])
    assert (R.ranks(only_misses.words(), 3, table, 1.0, 4) == 0).all()
    assert R.overflow_coverage(state_of(1, [1, 2, 2]).words()) == np.float32(2) / np.float32(3)


def test_coverage_is_the_rounded_float32_quotient():
    st = state_of(1, [1] * 7 + [None] * 3)                          # 7 / 10
    assert R.ranks(st.words(), 1, np.zeros(2, np.float32), 0.0, 2)[0, 1] == np.float32(np.float32(7) / np.float32(10))


def test_metadata_key_and_manifest():
    r = Renderer.__new__(Renderer)                                   # no device: only the name bookkeeping
    r.crypto_names, r.crypto_sphere = ["dragon.0", "dragon.1", "雲.2"], "sphere"
    md = r.cryptomatte_metadata()
    key = "%08x" % murmurhash3_32(b"CryptoObject", seed=0, positive=True)
    pre = f"cryptomatte/{key[:7]}/"
    assert set(md) == {pre + "name", pre + "hash", pre + "conversion", pre + "manifest"}
    assert md[pre + "name"] == "CryptoObject" and md[pre + "hash"] == "MurmurHash3_32" and md[pre + "conversion"] == "uint32_to_float32"
    man = json.loads(md[pre + "manifest"])
    assert set(man) == set(r.crypto_names) | {"sphere"}
    for name, hx in man.items():
        assert len(hx) == 8 and int(hx, 16) == R.id_bits(murmurhash3_32(name.encode("utf-8"), seed=0, positive=True))
    assert R.metadata_key("CryptoObject") == key[:7]
    assert list(r.cryptomatte_metadata("CryptoAsset"))[0].startswith("cryptomatte/" + R.metadata_key("CryptoAsset") + "/")


def test_bindings_and_refusals_without_a_device():
    assert N.VPT_CRYPTO_MAX_ENTRIES == R.MAX_ENTRIES == 32
    assert N.VPT_CRYPTO_SPHERE == R.SPHERE
    for name in ("vpt_set_cryptomatte", "vpt_cryptomatte_rank", "vpt_cryptomatte_hash"):
        assert name in N.EXPORTED_SYMBOLS
    assert V.lib.vpt_cryptomatte_hash.restype is C.c_uint32
    assert len(V.lib.vpt_cryptomatte_rank.argtypes) == 12
    assert V.lib.vpt_set_cryptomatte(None, None, 0) == -1
    assert V.lib.vpt_set_cryptomatte(None, C.c_void_p(0x1000), 8) == -1
    assert V.lib.vpt_cryptomatte_rank(None, 4, 4, C.c_void_p(0x1000), 4, None, 0, 0.0, 6, C.c_void_p(0x2000), None, None) == -1
