"""Every kernel launch goes through vgx_launch (csrc/vgx_internal.h), which counts it, attributes it to the open
profile scope's slot and checks its return code.  Outside that header's "kernel launches" section no source in
csrc/ may launch a kernel itself (<<<>>>, cudaLaunchKernelEx, cudaLaunchCooperativeKernel), read or clear the
runtime's last error, or write a launch count."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "voxgraph_b200", "csrc")
SECTION = re.compile(r"// -{20,} kernel launches\n.*?(?=// -{20,} )", re.S)
RULES = {
    "<<<>>> launch": re.compile(r"<<<"),
    "cudaLaunchKernelEx": re.compile(r"\bcudaLaunchKernelEx\b"),
    "cudaLaunchCooperativeKernel": re.compile(r"\bcudaLaunchCooperativeKernel\b"),
    "cudaGetLastError": re.compile(r"\bcudaGetLastError\b"),
    "write to a launch count": re.compile(r"(\.|->)\s*launches\s*(\+\+|--|[-+*/]?=(?!=))|(\+\+|--)\s*[\w.\->\[\]]*launches\b"),
}


def _code(text):
    """The text without comments; line numbers are kept."""
    text = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def _sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".h", ".cpp")):
            with open(os.path.join(CSRC, name)) as f:
                yield name, f.read()


def test_launch_helper_section_exists():
    with open(os.path.join(CSRC, "vgx_internal.h")) as f:
        section = SECTION.search(f.read())
    assert section, "vgx_internal.h has no kernel launches section"
    for what in ("int vgx_launch(", "cudaLaunchKernelEx", "cudaGetLastError", "struct VgxProfileScope"):
        assert what in section.group(0), what


def test_no_launch_bookkeeping_outside_the_helper():
    found = []
    for name, text in _sources():
        if name == "vgx_internal.h":   # blank the section out, keeping its lines
            text = SECTION.sub(lambda m: "\n" * m.group(0).count("\n"), text)
        for line_no, line in enumerate(_code(text).split("\n"), 1):
            found += ["%s:%d: %s: %s" % (name, line_no, rule, line.strip())
                      for rule, pattern in RULES.items() if pattern.search(line)]
    assert not found, "\n".join(found)
