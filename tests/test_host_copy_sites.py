"""Every copy between host and device, memset and stream synchronise goes through the helpers of the "host-device
copies" section of csrc/vgx_internal.h, which take element counts, run on the context's stream unless one is passed
and check their return codes.  Outside that section no source in csrc/ may call cudaMemcpy*, cudaMemset* or
cudaStreamSynchronize (cudaEventSynchronize stays allowed), and no call of a helper may work out a byte count with
sizeof."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "voxgraph_b200", "csrc")
SECTION = re.compile(r"// -{20,} host-device copies\n.*?(?=// -{20,} )", re.S)
RULES = {
    "cudaMemcpy*": re.compile(r"\bcudaMemcpy\w*"),
    "cudaMemset*": re.compile(r"\bcudaMemset\w*"),
    "cudaStreamSynchronize": re.compile(r"\bcudaStreamSynchronize\b"),
}
HELPER_CALL = re.compile(r"\bvgx_(upload|download|copy|read|fill)\s*\(")


def _code(text):
    """The text without comments; line numbers are kept."""
    text = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def _sources():
    """(name, code) of every source, the helper section blanked out with its lines kept."""
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".h", ".cpp")):
            with open(os.path.join(CSRC, name)) as f:
                text = f.read()
            if name == "vgx_internal.h":
                text = SECTION.sub(lambda m: "\n" * m.group(0).count("\n"), text)
            yield name, _code(text)


def _call_args(code, start):
    """The argument text of the call whose opening parenthesis is at code[start - 1]."""
    depth, i = 1, start
    while depth and i < len(code):
        depth += {"(": 1, ")": -1}.get(code[i], 0)
        i += 1
    return code[start:i - 1]


def test_copy_helper_section_exists():
    with open(os.path.join(CSRC, "vgx_internal.h")) as f:
        section = SECTION.search(f.read())
    assert section, "vgx_internal.h has no host-device copies section"
    for what in ("int vgx_upload(", "int vgx_download(", "int vgx_copy(", "int vgx_read(", "int vgx_fill(",
                 "int vgx_sync(", "void vgx_drain(", "cudaMemcpyAsync", "cudaMemsetAsync", "cudaStreamSynchronize"):
        assert what in section.group(0), what


def test_no_copies_outside_the_helpers():
    found = []
    for name, code in _sources():
        for line_no, line in enumerate(code.split("\n"), 1):
            found += ["%s:%d: %s: %s" % (name, line_no, rule, line.strip())
                      for rule, pattern in RULES.items() if pattern.search(line)]
    assert not found, "\n".join(found)


def test_helper_counts_are_elements():
    found = []
    for name, code in _sources():
        for m in HELPER_CALL.finditer(code):
            args = _call_args(code, m.end())
            if re.search(r"\bsizeof\b", args):
                line_no = code.count("\n", 0, m.start()) + 1
                found.append("%s:%d: vgx_%s(%s)" % (name, line_no, m.group(1), " ".join(args.split())))
    assert not found, "\n".join(found)
