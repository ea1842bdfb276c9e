"""Every ctypes declaration against the C++ compiler's view of its prototype: voxgraph_b200/_lib.py::SIGNATURES
against include/voxgraph_b200.h, oracle/oracle.py::SIGNATURES against oracle/vg_oracle.h and the oracle
harnesses' SIGNATURES against tests/oracle_harness.h; and every ctypes struct mirror of the oracle against its
typedef.  ctypes trusts argtypes blindly: a wrong width, signedness or argument count silently truncates a size or
reinterprets a float's bits.  No GPU and no built library: the driver only includes the header and describes
each prototype through decltype(&name), so nothing is linked against either library.

Rule: c_void_p matches any pointer except a pointer to a struct the header defines, which must be POINTER of that
struct's ctypes mirror (the driver static_asserts the exact typedef); POINTER(c_void_p) matches any
pointer-to-pointer; c_char_p matches char*.  Everything else must agree exactly: integer or float, width,
signedness, and the same for a pointer's pointee with const removed."""
import ctypes as C
import os
import subprocess

import support
from test_cabi_load import HEADER_STRUCTS

# the header typedef of every ctypes.Structure in oracle/oracle.py
ORACLE_STRUCTS = {"SolverOptions": "vgo_solver_options", "SolverSummary": "vgo_solver_summary",
                  "TsdfConfig": "vgo_tsdf_config", "EsdfConfig": "vgo_esdf_config", "TsdfStats": "vgo_tsdf_stats",
                  "TsdfTrace": "vgo_tsdf_trace", "Sampler": "vgo_sampler"}

DRIVER = r"""
#include <cstdio>
#include <string>
#include <tuple>
#include <type_traits>

template <class T, class = void> struct complete : std::false_type {};
template <class T> struct complete<T, std::void_t<decltype(sizeof(T))>> : std::true_type {};

template <class T> std::string describe() {
  if constexpr (std::is_void_v<T>) return "void";
  else if constexpr (std::is_pointer_v<T>) return "ptr(" + describe<std::remove_cv_t<std::remove_pointer_t<T>>>() + ")";
  else if constexpr (std::is_same_v<T, char>) return "char";
  else if constexpr (std::is_integral_v<T>) return (std::is_signed_v<T> ? "i" : "u") + std::to_string(8 * sizeof(T));
  else if constexpr (std::is_floating_point_v<T>) return "f" + std::to_string(8 * sizeof(T));
  else if constexpr (std::is_class_v<T>) return complete<T>::value ? "struct" : "opaque";
  else return "unknown";
}

template <class F> struct Sig;
template <class R, class... A> struct Sig<R (*)(A...)> {
  using ret = R;
  using args = std::tuple<A...>;
  static void print(const char* name) {
    std::printf("%s %s", name, describe<R>().c_str());
    (std::printf(" %s", describe<A>().c_str()), ...);
    std::printf("\n");
  }
};
template <class P> using pointee = std::remove_cv_t<std::remove_pointer_t<P>>;
"""


def describe(t):
    """A ctypes type in the driver's notation; "void*" and "ptr(ptr)" are the two wildcards of the rule."""
    if t is None:
        return "void"
    if t is C.c_void_p:
        return "void*"
    if t is C.c_char_p:
        return "ptr(char)"
    if t is C.c_char:
        return "char"
    if issubclass(t, C._Pointer):
        if issubclass(t._type_, C.Structure):
            return "ptr(struct)"
        return "ptr(ptr)" if t._type_ is C.c_void_p else "ptr(%s)" % describe(t._type_)
    if t in (C.c_float, C.c_double):
        return "f%d" % (8 * C.sizeof(t))
    if issubclass(t, C._SimpleCData) and isinstance(t(0).value, int):
        return ("i" if t(-1).value < 0 else "u") + str(8 * C.sizeof(t))
    raise TypeError("no rule for %r" % t)


def matches(py, c):
    if py == "void*":
        return c.startswith("ptr(") and c != "ptr(struct)"
    if py == "ptr(ptr)":
        return c.startswith("ptr(ptr(")
    return py == c


def driver_source(signatures, header, structs):
    """The driver: one line "name ret arg..." per entry, and a static_assert that every struct pointer's pointee is
    the typedef its mirror stands for (structs: {mirror name: typedef})."""
    lines = ['extern "C" {', '#include "%s"' % os.path.basename(header), "}", DRIVER]
    for name, (restype, argtypes) in signatures.items():
        for pos, t in [("ret", restype)] + list(enumerate(argtypes)):
            if isinstance(t, type) and issubclass(t, C._Pointer) and issubclass(t._type_, C.Structure):
                typedef = structs[t._type_.__name__]
                where = ("Sig<decltype(&%s)>::ret" % name if pos == "ret" else
                         "std::tuple_element_t<%d, Sig<decltype(&%s)>::args>" % (pos, name))
                lines.append('static_assert(std::is_same_v<pointee<%s>, %s>, "%s, %s: not a %s*");'
                             % (where, typedef, name, "return type" if pos == "ret" else "argument %d" % pos, typedef))
    lines.append("int main() {")
    lines += ['  Sig<decltype(&%s)>::print("%s");' % (name, name) for name in signatures]
    lines += ["  return 0;", "}"]
    return "\n".join(lines)


def header_prototypes(tmp_path, signatures, header, structs, include_dirs=()):
    """{name: [ret, arg...]} in the driver's notation, from the compiled driver."""
    src = tmp_path / "signatures.cpp"
    src.write_text(driver_source(signatures, header, structs))
    exe = tmp_path / "signatures"
    inc = ["-I" + d for d in (os.path.dirname(header),) + tuple(include_dirs)]
    p = subprocess.run(["g++", "-std=c++17"] + inc + [str(src), "-o", str(exe)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout
    out = subprocess.run([str(exe)], check=True, stdout=subprocess.PIPE, text=True).stdout
    return {line.split()[0]: line.split()[1:] for line in out.splitlines()}


def mismatches(tmp_path, signatures, header, structs, include_dirs=()):
    """"name: ctypes (...), header (...)" for every entry whose declaration does not match its prototype."""
    protos = header_prototypes(tmp_path, signatures, header, structs, include_dirs)
    bad = []
    for name, (restype, argtypes) in signatures.items():
        c = protos[name]
        py = [describe(restype)] + [describe(t) for t in argtypes]
        if len(py) != len(c) or not all(matches(a, b) for a, b in zip(py, c)):
            bad.append("%s: ctypes (%s), header (%s)" % (name, ", ".join(py), ", ".join(c)))
    return bad


def test_every_signature_matches_the_header(tmp_path):
    from voxgraph_b200 import _lib
    assert set(_lib.SIGNATURES) == support.header_functions(), "an entry missing from SIGNATURES, or an extra one"
    bad = mismatches(tmp_path, _lib.SIGNATURES, support.LIBRARY_HEADER, HEADER_STRUCTS)
    assert not bad, "\n".join(bad)


def test_every_oracle_signature_matches_the_header(tmp_path):
    from oracle import oracle as o
    assert set(o.SIGNATURES) == support.header_functions(support.ORACLE_HEADER, "vgo_"), \
        "an entry missing from oracle.SIGNATURES, or an extra one"
    bad = mismatches(tmp_path, o.SIGNATURES, support.ORACLE_HEADER, ORACLE_STRUCTS)
    assert not bad, "\n".join(bad)


def test_every_oracle_harness_signature_matches_the_header(tmp_path):
    import project_colour_oracle
    import project_oracle
    import transform_oracle
    signatures = {**project_oracle.SIGNATURES, **project_colour_oracle.SIGNATURES, **transform_oracle.SIGNATURES}
    assert set(signatures) == support.header_functions(support.HARNESS_HEADER, "(?:vgp|vgpc|vgt)_"), \
        "a harness function missing from its loader's SIGNATURES, or an extra one"
    bad = mismatches(tmp_path, signatures, support.HARNESS_HEADER, ORACLE_STRUCTS,
                     [os.path.dirname(support.ORACLE_HEADER)])
    assert not bad, "\n".join(bad)


def test_oracle_struct_layouts_match_header(tmp_path):
    from oracle import oracle as o
    support.check_struct_layouts(tmp_path, o, ORACLE_STRUCTS, support.ORACLE_HEADER)
