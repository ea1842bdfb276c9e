"""Submap collection streams on the host (no GPU): vgx_collection_scan reads the committed fixtures
(tests/golden/collection_*.bin, serialised by Google's protobuf runtime) as the .npz describes them,
and refuses every malformed framing with VGX_ERR_INVALID.  The malformations are built here by a
small independent encoder (collection_stream.py) that first has to reproduce the unpacked fixture byte
for byte."""
import ctypes as C
import os

import numpy as np
import pytest

from collection_stream import CASES, GOLDEN, build as _build, boundaries as _boundaries, read as _read, varint as _varint
from voxgraph_b200 import _lib

INVALID, CAPACITY = _lib.VGX_ERR_INVALID, _lib.VGX_ERR_CAPACITY


@pytest.fixture(scope="module")
def lib():
    from voxgraph_b200 import build, _lib
    build.build()
    return _lib.load()


@pytest.fixture(scope="module")
def expected():
    return dict(np.load(os.path.join(GOLDEN, "collection_expected.npz")))


def _scan_rc(lib, data):
    from voxgraph_b200 import _lib
    n = C.c_int(0)
    out = (_lib.CollectionEntry * 16)()
    return lib.vgx_collection_scan(data, len(data), 16, out, C.byref(n))


# ---------------------------------------------------------------- tests
@pytest.mark.parametrize("case", CASES)
def test_scan_matches_fixture(lib, expected, case):
    from voxgraph_b200 import api
    entries = api.Context.collection_scan(_read(case))
    assert [e["id"] for e in entries] == expected["ids"].tolist()
    assert [e["num_blocks"] for e in entries] == expected["num_blocks"].tolist()
    for k, e in enumerate(entries):
        assert e["voxel_size"] == expected["voxel_size"] and e["voxels_per_side"] == expected["vps"]
        assert np.array_equal(e["T_M_S"].view(np.uint32), expected["poses"][k].view(np.uint32))


def test_scan_empty_collection(lib):
    from voxgraph_b200 import api
    assert api.Context.collection_scan(_read("empty")) == []


def test_scan_capacity(lib):
    from voxgraph_b200 import _lib
    data = _read("unpacked")
    n = C.c_int(0)
    out = (_lib.CollectionEntry * 2)()
    assert lib.vgx_collection_scan(data, len(data), 2, out, C.byref(n)) == CAPACITY and n.value == 3
    assert lib.vgx_collection_scan(data, len(data), 0, None, C.byref(n)) == CAPACITY and n.value == 3


def test_independent_encoder_reproduces_fixture(expected):
    assert _build(expected) == _read("unpacked")


def test_truncation_rejected(lib):
    data = _read("unpacked")
    cuts = set()
    for s in _boundaries(data):
        cuts.update({s, s + 1, s + 2, s + 5, s + 12})   # at the boundary, in the length, in the first fields
    for cut in sorted(c for c in cuts if c < len(data)):
        assert _scan_rc(lib, data[:cut]) == INVALID, cut
    assert _scan_rc(lib, b"") == INVALID


def test_overlong_varints_rejected(lib):
    data = _read("unpacked")
    n0 = data[0]
    assert n0 < 0x80
    six = bytes([n0 | 0x80, 0x80, 0x80, 0x80, 0x80, 0x00])     # the header length in 6 bytes
    assert _scan_rc(lib, six + data[1:]) == INVALID
    five = bytes([n0 | 0x80, 0x80, 0x80, 0x80, 0x00])          # 5 bytes is still a valid varint
    assert _scan_rc(lib, five + data[1:]) == 0
    wide = bytes([n0 | 0x80, 0x80, 0x80, 0x80, 0x10])          # a 33-bit length
    assert _scan_rc(lib, wide + data[1:]) == INVALID


def test_overlong_field_value_rejected(lib, expected):
    # num_submaps written as a 6-byte varint: the header message grows by 5 bytes
    hdr_len = _read("unpacked")[0]
    data = _read("unpacked")[1:]
    hdr, rest = data[:hdr_len], data[hdr_len:]
    k = hdr.index(b"\x18")   # field 3, varint
    assert hdr[k + 1] == 3
    bad = hdr[:k + 1] + bytes([0x83, 0x80, 0x80, 0x80, 0x80, 0x00]) + hdr[k + 2:]
    assert _scan_rc(lib, _varint(len(bad)) + bad + rest) == INVALID


KNOWN_FIELDS = ["header.1", "header.2", "header.3", "submap.1", "submap.2", "submap.3", "transform.1",
                "transform.2", "position.1", "position.2", "position.3", "rotation.1", "rotation.2",
                "rotation.3", "rotation.4", "block.1", "block.2", "block.3", "block.4", "block.5", "block.6",
                "block.7"]
NATURAL = {"header.1": 1, "header.2": 0, "header.3": 0, "submap.1": 0, "submap.2": 0, "submap.3": 2,
           "transform.1": 2, "transform.2": 2, "block.1": 0, "block.6": 0, "block.7": 0}


@pytest.mark.parametrize("field", KNOWN_FIELDS)
def test_wrong_wire_type_rejected(lib, expected, field):
    natural = NATURAL.get(field, 1)
    for wire in (0, 1, 2, 5):
        if wire == natural or (field == "block.7" and wire == 2):   # voxel_data may be packed
            continue
        assert _scan_rc(lib, _build(expected, over={field: wire})) == INVALID, (field, wire)


def test_counts_off_by_one_rejected(lib, expected):
    n, nb = len(expected["ids"]), int(expected["num_blocks"][0])
    assert _scan_rc(lib, _build(expected)) == 0
    for bad in (dict(num_submaps=n - 1), dict(num_submaps=n + 1), dict(num_blocks=nb - 1),
                dict(num_blocks=nb + 1)):
        assert _scan_rc(lib, _build(expected, **bad)) == INVALID, bad


def test_trailing_bytes_rejected(lib):
    data = _read("unpacked")
    assert _scan_rc(lib, data + b"\x00") == INVALID
    assert _scan_rc(lib, data + data[:data[0] + 1]) == INVALID   # one more delimited message


def test_block_geometry_must_match_header(lib, expected):
    vps, vs = int(expected["vps"]), float(expected["voxel_size"])
    assert _scan_rc(lib, _build(expected, block_vps=vps * 2)) == INVALID
    assert _scan_rc(lib, _build(expected, block_voxel_size=0.2)) == INVALID   # the double, not the float
    assert _scan_rc(lib, _build(expected, block_voxel_size=vs)) == 0
