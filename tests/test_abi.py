"""CPU tests: the C-ABI library loads and exports every symbol declared in include/metamorph_b200.h;
argument validation fails loudly without touching a GPU."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "metamorph_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mm_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_declared_symbols():
    from metamorph_b200 import _build
    from metamorph_b200._lib import lib
    _build.build(verbose=False)
    l = lib()
    names = _declared()
    assert len(names) >= 35
    missing = [n for n in names if not hasattr(l, n)]
    assert not missing, f"declared but not exported: {missing}"
    assert l.mm_abi_version() == 1


def test_header_compiles_as_c():
    import subprocess
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write('#include "metamorph_b200.h"\nint main(void){return 0;}\n')
        subprocess.run(["gcc", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", c],
                       check=True)


def test_bad_arguments_fail_loudly_without_gpu():
    from metamorph_b200._lib import MetaMorphB200Error, call, ll
    from ctypes import c_float, c_int, c_void_p
    with pytest.raises(MetaMorphB200Error, match="H%8"):
        call("mm_rmsnorm_fwd", c_void_p(0), c_void_p(0), c_void_p(0), ll(4), ll(7), c_float(1e-5), c_void_p(0))
    with pytest.raises(MetaMorphB200Error, match="batch"):
        call("mm_skinny_gemm", c_void_p(0), c_void_p(0), c_void_p(0), c_void_p(0), c_void_p(0), ll(64), ll(64),
             ll(64), ll(0), c_int(33), c_int(64), c_int(64), c_int(0), c_int(0), c_void_p(0))
    a = c_void_p(256)   # aligned, never dereferenced: the tile-width check rejects the call first
    with pytest.raises(MetaMorphB200Error, match="force_bn"):
        call("mm_gemm_bf16", a, a, a, c_void_p(0), c_void_p(0), c_void_p(0), ll(128), ll(128), ll(128), ll(128),
             ll(128), ll(128), ll(0), ll(0), c_int(0), c_int(0), c_int(0), c_int(0), c_int(0), c_float(1.0), c_int(512),
             c_void_p(0))


def test_product_never_imports_oracle():
    bad = []
    for dp, _, files in os.walk(os.path.join(ROOT, "metamorph_b200")):
        for f in files:
            if f.endswith(".py") and re.search(r"^\s*(from|import)\s+oracle", open(os.path.join(dp, f)).read(), flags=re.M):
                bad.append(os.path.join(dp, f))
    assert not bad, f"product code must not import the oracle: {bad}"


def test_ctypes_call_sites_pass_the_declared_number_of_arguments():
    """ctypes does not check arity: every `call("mm_x", ...)` / `lib().mm_x(...)` in the package must pass exactly as
    many arguments as the prototype in include/metamorph_b200.h declares (a mismatch would be undefined behaviour on
    the GPU box, not an exception)."""
    import ast
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "metamorph_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(mm_\w+)\s*\(([^;{]*?)\)\s*;", header, flags=re.S):
        params = m.group(2).strip()
        protos[m.group(1)] = 0 if params in ("", "void") else params.count(",") + 1
    assert len(protos) >= 40
    checked = 0
    pkg = os.path.join(root, "metamorph_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if not f.endswith(".py"):
                continue
            tree = ast.parse(open(os.path.join(dirpath, f)).read())
            for node in ast.walk(tree):
                if not isinstance(node, ast.Call):
                    continue
                name, nargs = None, None
                if isinstance(node.func, ast.Name) and node.func.id == "call" and node.args and \
                        isinstance(node.args[0], ast.Constant) and isinstance(node.args[0].value, str):
                    name, nargs = node.args[0].value, len(node.args) - 1
                elif isinstance(node.func, ast.Name) and node.func.id == "call" and node.args and \
                        isinstance(node.args[0], ast.IfExp):
                    # call("a" if cond else "b", ...): both names must agree with the argument count
                    for branch in (node.args[0].body, node.args[0].orelse):
                        if isinstance(branch, ast.Constant) and branch.value in protos:
                            assert protos[branch.value] == len(node.args) - 1, (f, branch.value)
                            checked += 1
                    continue
                if name is None or any(isinstance(a, ast.Starred) for a in node.args):
                    continue
                assert name in protos, f"{f}: {name} is not declared in the header"
                assert protos[name] == nargs, f"{f}: {name} declared with {protos[name]} parameters, called with {nargs}"
                checked += 1
    assert checked >= 35
