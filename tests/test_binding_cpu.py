"""The ctypes mirror of include/sbi_b200.h in `sbi_b200._lib` against the header itself: every struct's size and
field offsets and every shared integer constant, as a C++ probe compiled against the header reports them, and
every prototype's parameter count and stream parameter.  A drifted layout or constant would make every kernel read
garbage without any error, so this is checked without the library or a GPU."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from sbi_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "sbi_b200.h")


def _header_text() -> str:
    with open(HEADER) as f:
        src = f.read()
    return re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", src, flags=re.S))


def _structs():
    """{ctypes struct: its C typedef}: `NsfModel` mirrors `sbi_nsf_model`, `Lc2stNet` `sbi_lc2st_net`, ..."""
    out = {}
    for name, v in vars(_lib).items():
        if isinstance(v, type) and issubclass(v, C.Structure) and v.__module__ == _lib.__name__:
            out[v] = "sbi_" + re.sub(r"(?<!^)(?=[A-Z])", "_", name).lower()
    return out


def _constants(hdr: str):
    """{name in _lib: name in the header} of the integer constants the header also defines (`L_BLK0` is
    `SBI_L_BLK0`, `SBI_HMC_NV0` itself)."""
    out = {}
    for name, v in vars(_lib).items():
        if re.fullmatch(r"[A-Z][A-Z0-9_]*", name) and isinstance(v, int) and not isinstance(v, bool):
            c_name = name if name.startswith("SBI_") else "SBI_" + name
            if re.search(rf"\b{c_name}\b", hdr):
                out[name] = c_name
    return out


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    """{key: value} printed by a C++ program built against the header: ("size", struct), ("offset", struct,
    field) and ("const", name)."""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    lines = []
    for cls, c_name in _structs().items():
        lines.append(f'  std::printf("size {cls.__name__} %zu\\n", sizeof({c_name}));')
        for field, *_ in cls._fields_:
            lines.append(f'  std::printf("offset {cls.__name__} {field} %zu\\n", offsetof({c_name}, {field}));')
    for name, c_name in _constants(_header_text()).items():
        lines.append(f'  std::printf("const {name} %lld\\n", (long long)({c_name}));')
    d = tmp_path_factory.mktemp("abi_probe")
    (d / "probe.cpp").write_text('#include <cstddef>\n#include <cstdio>\n#include "sbi_b200.h"\n'
                                 "int main() {\n" + "\n".join(lines) + "\n  return 0;\n}\n")
    subprocess.run([cxx, "-std=c++17", "-I", os.path.dirname(HEADER), str(d / "probe.cpp"), "-o", str(d / "probe")],
                   check=True, capture_output=True, text=True)
    out = subprocess.run([str(d / "probe")], check=True, capture_output=True, text=True).stdout
    return {tuple(line.split()[:-1]): int(line.split()[-1]) for line in out.splitlines()}


def test_struct_layouts_match_the_header(probe):
    structs = _structs()
    assert len(structs) >= 15, sorted(c.__name__ for c in structs)
    for cls in structs:
        assert C.sizeof(cls) == probe[("size", cls.__name__)], f"sizeof {cls.__name__}"
        for field, *_ in cls._fields_:
            assert getattr(cls, field).offset == probe[("offset", cls.__name__, field)], f"{cls.__name__}.{field}"


def test_constants_match_the_header(probe):
    consts = _constants(_header_text())
    assert len(consts) >= 60, sorted(consts)
    for name in consts:
        assert getattr(_lib, name) == probe[("const", name)], name


def test_prototypes_match_the_header():
    """Every entry point has the header's parameter count and carries the stream marker (`call` launches it) exactly
    when its last parameter is `void* stream`."""
    declared = {}
    for m in re.finditer(r"\b(sbi_b200_\w+)\s*\(([^()]*)\)\s*;", _header_text()):
        params = [p.strip() for p in m.group(2).split(",")]
        declared[m.group(1)] = [] if params == ["void"] else params
    assert set(declared) == set(_lib.exported_symbols())
    n_stream = 0
    for name, (_, argtypes) in _lib._EXPORTS.items():
        params = declared[name]
        assert len(argtypes) == len(params), name
        takes_stream = bool(params) and re.fullmatch(r"void\s*\*\s*stream", params[-1]) is not None
        assert (bool(argtypes) and argtypes[-1] is _lib._Stream) == takes_stream, name
        n_stream += takes_stream
    assert n_stream == len(_lib._LAUNCH) > 0
