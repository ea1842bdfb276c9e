"""Device memory has one owner and scratch has one layout call (voxgraph_b200/csrc).

VgxBuffer in vgx_internal.h is the only code that allocates or frees device and pinned host memory;
p2p.cu keeps its own peer-exchange region, which is exported to other processes.  The scratch arenas
of vgx_ctx are laid out only by vgx_carve, so no pass computes offsets into one by hand and a pass
cannot keep a pointer into an arena without going through the layout call."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "voxgraph_b200", "csrc")
OWNER = "vgx_internal.h"
ARENAS = ("d_scratch", "d_work", "d_work2", "h_pinned")


def _sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".h", ".cpp")):
            with open(os.path.join(CSRC, name)) as f:
                yield name, f.read()


def test_only_the_owner_allocates_and_frees():
    calls = re.compile(r"\bcuda(Malloc|MallocHost|Free|FreeHost)\b")
    found = {name: sorted(set(calls.findall(src))) for name, src in _sources()
             if name not in (OWNER, "p2p.cu") and calls.search(src)}
    assert found == {}, "allocations outside VgxBuffer: %s" % found


def test_arenas_are_read_only_through_vgx_carve():
    mention = re.compile(r"->(%s)\b" % "|".join(ARENAS))
    carved = re.compile(r"\bvgx_carve\(\s*\w+,\s*\w+->(%s)," % "|".join(ARENAS))
    direct = {}
    for name, src in _sources():
        if name == OWNER:
            continue
        n = len(mention.findall(src)) - len(carved.findall(src))
        if n:
            direct[name] = n
    assert direct == {}, "arena members used outside vgx_carve: %s" % direct


def test_no_hand_written_layout_arithmetic():
    hand = re.compile(r"\+ 255\) & ~|\balign256\b")
    found = [name for name, src in _sources() if name != OWNER and hand.search(src)]
    assert found == [], "256-byte rounding outside vgx_carve: %s" % found
    owner = dict(_sources())[OWNER]
    assert len(hand.findall(owner)) == 1 and "align256" not in owner
