"""Every kernel finds a voxel in a layer's bricks through the helpers of the "brick addressing" section of
csrc/layer_access.cuh: voxel index to slot and voxel, slot and voxel to address, voxel counts, voxel centres and
the split of a global voxel index into block and voxel.  Outside that section no source in csrc/ may shift by a
brick's voxel count (<< or >> by 3 * sh or 2 * sh), mask a voxel index with vps - 1, or write a voxel centre
(+ 0.5f) * voxel_size.  The registration path (registration.cu, registration.cuh) keeps its own addressing, which
is specialised for 16-voxel bricks."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "voxgraph_b200", "csrc")
SECTION = re.compile(r"// -{20,} brick addressing\n.*?(?=// -{20,} )", re.S)
EXEMPT = ("registration.cu", "registration.cuh")
RULES = {
    "brick shift": re.compile(r"(<<|>>)\s*\(\s*[23]\s*\*\s*[\w.>\-]*\bsh\)"),
    "voxel mask": re.compile(r"&\s*\(\s*[\w.>\-]*\bvps\s*-\s*1\s*\)"),
    "voxel centre": re.compile(r"\+\s*0\.5f\s*\)\s*\*\s*[\w.>\-]*\bvoxel_size\b"),
}


def _code(text):
    """The text without comments; line numbers are kept."""
    text = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def test_addressing_section_exists():
    with open(os.path.join(CSRC, "layer_access.cuh")) as f:
        section = SECTION.search(f.read())
    assert section, "layer_access.cuh has no brick addressing section"
    for what in ("bool vgx_vps_ok(", "size_t vgx_voxel_count(", "size_t vgx_voxel_index(", "int vgx_voxel_of(",
                 "float vgx_voxel_centre(", "bool vgx_global_block(", "void vgx_forward_slots("):
        assert what in section.group(0), what


def test_no_voxel_addressing_outside_the_helpers():
    found = []
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith((".cu", ".cuh", ".h", ".cpp")) or name in EXEMPT:
            continue
        with open(os.path.join(CSRC, name)) as f:
            text = f.read()
        if name == "layer_access.cuh":   # blank the section out, keeping its lines
            text = SECTION.sub(lambda m: "\n" * m.group(0).count("\n"), text)
        for line_no, line in enumerate(_code(text).split("\n"), 1):
            found += ["%s:%d: %s: %s" % (name, line_no, rule, line.strip())
                      for rule, pattern in RULES.items() if pattern.search(line)]
    assert not found, "\n".join(found)
