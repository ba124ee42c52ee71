"""The ctypes mirrors of api.py against include/hunter_b200.h (no GPU, no built library). Every `typedef struct { ... } hb_x;` of the header
has a mirror HbX with the layout the C++ compiler gives the struct: size, alignment, field names in order, and per field its offset, size,
element size, element kind (floating, signed, unsigned, struct) and array extents. A wrong mirror does not fail a call: the library reads
the wrong bytes. The Python constants that restate numeric macros of the header have their values."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from hunter_bipedal_control_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = re.sub(r"/\*.*?\*/|//[^\n]*", " ", open(os.path.join(ROOT, "include", "hunter_b200.h")).read(), flags=re.S)   # without comments


def _struct_fields(body):
    """[(name, base type)] of the declarations of a struct body, multi-declarators (`double merit0, merit1;`) included."""
    fields = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        base, declarators = decl.split(None, 1)
        fields += [(re.match(r"\s*(\w+)", d).group(1), base) for d in declarators.split(",")]
    return fields


STRUCTS = {name: _struct_fields(body) for body, name in re.findall(r"typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;", HEADER, re.S)}
MACROS = {k: int(v) for k, v in re.findall(r"^\s*#define\s+(HB_\w+)\s+(\d+)\s*$", HEADER, re.M)}
PY_CONSTANTS = ["HB_MAX_EVENTS", "HB_MAX_HORIZON", "HB_MAX_TARGETS", "HB_MAX_SEGMENTS", "HB_HOQP_MAX_LEVELS", "HB_HOQP_N", "HB_HOQP_MAX_EQ", "HB_HOQP_MAX_IN",
                "HB_HOQP_MAX_STACKED", "HB_ACT_CAPACITY", "HB_ROLLOUT_MAX_CMDS", "HB_MAX_PUSHES"]

PROBE = r"""#include "hunter_b200.h"
#include <cstddef>
#include <cstdio>
#include <type_traits>
template <class F> void extents() {
  if constexpr (std::rank_v<F> > 0) {
    std::printf(" %zu", std::extent_v<F>);
    extents<std::remove_extent_t<F>>();
  }
}
template <class F> void field(const char* s, const char* f, std::size_t offset) {
  using E = std::remove_all_extents_t<F>;
  std::printf("field %s %s %zu %zu %zu %c", s, f, offset, sizeof(F), sizeof(E),
              std::is_floating_point_v<E> ? 'f' : std::is_signed_v<E> ? 'i' : std::is_unsigned_v<E> ? 'u' : 'V');
  extents<F>();
  std::printf("\n");
}
int main() {
@BODY@
}
"""


def _mirror_name(c_name):
    return "".join(w.capitalize() for w in c_name.split("_"))          # hb_sim_params -> HbSimParams


def _element(t):
    """ctypes field type -> (element type, array extents)."""
    shape = []
    while issubclass(t, C.Array):
        shape.append(t._length_)
        t = t._type_
    return t, tuple(shape)


def _mirror_layout(T):
    fields = []
    for name, t in T._fields_:
        e, shape = _element(t)
        fields.append((name, getattr(T, name).offset, getattr(T, name).size, C.sizeof(e), np.dtype(e).kind, shape))
    return dict(size=C.sizeof(T), align=C.alignment(T), fields=fields)


@pytest.fixture(scope="module")
def c_layout(tmp_path_factory):
    """{C name: dict(size, align, fields)} as g++ lays out the header's structs, in _mirror_layout's form."""
    body = []
    for s, fields in STRUCTS.items():
        body.append('  std::printf("struct %s %%zu %%zu\\n", sizeof(%s), alignof(%s));' % (s, s, s))
        body += ['  field<decltype(%s::%s)>("%s", "%s", offsetof(%s, %s));' % (s, f, s, f, s, f) for f, _ in fields]
    d = tmp_path_factory.mktemp("abi_layout")
    (d / "probe.cpp").write_text(PROBE.replace("@BODY@", "\n".join(body)))
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", str(d / "probe"), str(d / "probe.cpp")],
                   check=True)
    layout = {}
    for line in subprocess.run([str(d / "probe")], check=True, capture_output=True, text=True).stdout.splitlines():
        tok = line.split()
        if tok[0] == "struct":
            layout[tok[1]] = dict(size=int(tok[2]), align=int(tok[3]), fields=[])
        else:
            layout[tok[1]]["fields"].append((tok[2], int(tok[3]), int(tok[4]), int(tok[5]), tok[6], tuple(int(x) for x in tok[7:])))
    return layout


def test_header_parse_finds_every_struct():
    assert len(STRUCTS) == len(re.findall(r"typedef\s+struct\s*\{", HEADER)) >= 22
    assert all(STRUCTS.values())


@pytest.mark.parametrize("name", sorted(STRUCTS))
def test_struct_mirror_matches_the_header(name, c_layout):
    mirror = getattr(api, _mirror_name(name), None)
    assert mirror is not None, "%s has no ctypes mirror %s in api.py" % (name, _mirror_name(name))
    py, c = _mirror_layout(mirror), c_layout[name]
    assert [f[0] for f in py["fields"]] == [f for f, _ in STRUCTS[name]]
    assert py == c
    for (f, base), (_, t) in zip(STRUCTS[name], mirror._fields_):          # a struct-typed field holds the mirror of its C type
        if issubclass(_element(t)[0], C.Structure):
            assert _element(t)[0] is getattr(api, _mirror_name(base)), (name, f)


def test_constants_match_the_header():
    py = {k: v for k, v in vars(api).items() if k.startswith("HB_")}
    assert set(PY_CONSTANTS) <= set(py)
    assert py == {k: MACROS.get(k) for k in py}
    assert api.ROLLOUT_FAIL == {k[len("HB_ROLLOUT_FAIL_"):].lower(): v for k, v in MACROS.items() if k.startswith("HB_ROLLOUT_FAIL_")}
