"""The ctypes binding is parsed from include/fgt_b200.h (fgt_b200/lib.py). These tests tie the parse to the library's
definitions, to the C compiler's struct layout and to every `lib.call` in the package."""
import ast
import ctypes
import glob
import os
import re
import shutil
import subprocess

import pytest
import torch

from fgt_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CC = next((c for c in ("cc", "gcc", "clang") if shutil.which(c)), None)


def test_every_definition_has_a_parsed_prototype():
    """The parser missed no prototype: its entries are the library's extern "C" definitions (fgt_debug_* switches are
    undeclared on purpose)."""
    defined = set()
    for path in glob.glob(os.path.join(ROOT, "fgt_b200", "csrc", "*.cu")):
        with open(path) as f:
            defined |= set(re.findall(r'extern\s+"C"\s+[^;{}()]*?\b(fgt_\w+)\s*\(', f.read()))
    assert {n for n in defined if not n.startswith("fgt_debug_")} == set(lib.PROTOS)


@pytest.mark.skipif(CC is None, reason="no C compiler")
def test_struct_layout_matches_the_c_compiler(tmp_path):
    """sizeof and every field's offsetof of the descriptor structs, compiled from the header, equal the ctypes layout."""
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "fgt_b200.h"', "int main(void) {"]
    want = []
    for s in (lib.FgtASeg, lib.FgtGemmDesc, lib.FgtAttnDesc):
        lines.append(f'printf("%zu\\n", sizeof({s.__name__}));')
        want.append(ctypes.sizeof(s))
        for f, _ in s._fields_:
            lines.append(f'printf("%zu\\n", offsetof({s.__name__}, {f}));')
            want.append(getattr(s, f).offset)
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines + ["return 0;", "}"]))
    subprocess.run([CC, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert [int(x) for x in got] == want


def test_kernels_launch_only_through_the_checked_launcher():
    """Launches, the dynamic shared-memory opt-in and grid-stride sizing live in common.h / common.cu: no other source
    launches a kernel, reads the runtime's last error, sets a kernel attribute or sizes a grid-stride grid itself."""
    banned = ("cudaLaunchKernelEx", "cudaFuncSetAttribute", "cudaGetLastError", "<<<", "launch_k(", "num_sms()) * 16",
              "num_sms() * 16")
    csrc = os.path.join(ROOT, "fgt_b200", "csrc")
    paths = glob.glob(os.path.join(csrc, "*.cu")) + glob.glob(os.path.join(csrc, "*.cuh"))
    assert len(paths) > 10
    for path in paths:
        if os.path.basename(path) == "common.cu":
            continue
        with open(path) as f:
            src = f.read()
        found = [b for b in banned if b in src]
        assert not found, (os.path.basename(path), found)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the launch errors of a host without a CUDA device")
def test_launch_errors_name_the_kernel_without_a_device():
    """With no device the runtime refuses every launch before any pointer is used. Each entry returns FGT_ERR_CUDA
    with an error naming its own kernel, from its own launch (im2col_nchw: from its shared-memory opt-in), not an
    error an earlier call left pending."""
    L = lib.load()
    p = ctypes.c_void_p(1 << 20)                    # aligned, never dereferenced
    ll, f32 = ctypes.c_longlong, ctypes.c_float
    calls = [
        (L.fgt_avgpool2, (p, ll(1), 4, 4, p, None), "avgpool2_kernel"),
        (L.fgt_plane_max, (p, 1, ll(16), p, None), "plane_max_kernel"),
        (L.fgt_im2col_nchw, (p, 4, None, 0, 1, 8, 8, 3, 1, 1, 0, 8, 8, 64, f32(1), f32(0), p, ll(0), None),
         "im2col_nchw_kernel"),
    ]
    for fn, args, kernel in calls * 2:
        assert fn(*args) == lib.ERR_CUDA, fn.__name__
        assert kernel in L.fgt_last_error().decode(), (fn.__name__, L.fgt_last_error())


def _calls():
    """(module, line, entry, positional argument count) of every `lib.call` under fgt_b200/. A starred argument must be
    a tuple literal assigned in the same module."""
    for path in sorted(glob.glob(os.path.join(ROOT, "fgt_b200", "*.py"))):
        with open(path) as f:
            tree = ast.parse(f.read())
        tuples = {t.id: len(n.value.elts) for n in ast.walk(tree) if isinstance(n, ast.Assign)
                  and isinstance(n.value, ast.Tuple) for t in n.targets if isinstance(t, ast.Name)}
        for n in ast.walk(tree):
            if isinstance(n, ast.Call) and ast.unparse(n.func) in ("lib.call", "call"):
                where = f"{os.path.basename(path)}:{n.lineno}"
                assert isinstance(n.args[0], ast.Constant), f"{where}: the entry must be a literal"
                count = sum(tuples[a.value.id] if isinstance(a, ast.Starred) else 1 for a in n.args[1:])
                assert all(k.arg == "kernels" for k in n.keywords), where
                yield where, n.args[0].value, count


def test_every_call_names_an_entry_with_its_parameter_count():
    calls = list(_calls())
    assert len(calls) > 60
    for where, name, count in calls:
        assert name in lib.PROTOS, f"{where}: {name} is not declared in the header"
        p = lib.PROTOS[name]
        assert count == len(p.names) - p.stream, f"{where}: {name} takes {p.names}, called with {count} arguments"


def test_parser_handles_the_header_forms_and_refuses_unknown_types():
    structs, enums, protos = lib.parse_header("""
        /* comment: int fgt_not_a_prototype(int x); */
        typedef struct { int a, b; long long c; } P;   // comma declarators
        typedef struct { P p[2]; const float* q; } Q;  /* a nested struct array */
        enum { FGT_X = -1, FGT_Y };
        long long fgt_size(int n, const unsigned char h[64], void** out, fgt_stream_t stream);
        const char* fgt_msg(void);""")
    assert [f for f, _ in structs["P"]._fields_] == ["a", "b", "c"] and ctypes.sizeof(structs["Q"]) == 40
    assert enums == {"FGT_X": -1, "FGT_Y": 0}
    assert set(protos) == {"fgt_size", "fgt_msg"}
    p = protos["fgt_size"]
    assert p.restype is ctypes.c_longlong and p.stream and p.names == ["n", "h", "out", "stream"]
    assert p.argtypes == [ctypes.c_int] + [ctypes.c_void_p] * 3
    assert protos["fgt_msg"].restype is ctypes.c_char_p and protos["fgt_msg"].argtypes == []
    with pytest.raises(ValueError, match="unsigned short"):
        lib.parse_header("int fgt_x(unsigned short n, fgt_stream_t stream);")
    with pytest.raises(ValueError, match="bool on"):
        lib.parse_header("typedef struct { bool on; } S;")
    with pytest.raises(ValueError, match="void fgt_y"):
        lib.parse_header("void fgt_y(int a);")
