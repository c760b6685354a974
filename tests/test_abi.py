"""CPU: the C-ABI library loads without a GPU and exports exactly the symbols include/dsvg_b200.h declares; the ctypes
signature table matches the header's argument counts."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    hdr = open(os.path.join(ROOT, "include", "dsvg_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    out = {}
    for m in re.finditer(r"\b(?:int|const char\*|unsigned long long)\s+(dsvg_[a-z0-9_]+)\s*\(([^;]*?)\)\s*;", hdr, re.S):
        args = m.group(2).strip()
        out[m.group(1)] = 0 if args == "void" else len(args.split(","))
    return out


def test_library_exports_every_declared_symbol():
    from deepsvg_b200 import _lib
    lib = _lib.load()
    fns = _header_functions()
    assert len(fns) >= 28
    for name in fns:
        assert hasattr(lib, name), name
    assert lib.dsvg_abi_version() == 6
    assert lib.dsvg_launch_count() == 0          # nothing launched: loading needs no GPU


def test_ctypes_table_matches_header():
    from deepsvg_b200._abi import SIGNATURES
    fns = _header_functions()
    assert set(SIGNATURES) == set(fns) - {"dsvg_last_error", "dsvg_launch_count"}
    for name, (_, argtypes) in SIGNATURES.items():
        assert len(argtypes) == fns[name], name


def test_epilogue_struct_matches_header():
    from deepsvg_b200._lib import Epilogue
    hdr = open(os.path.join(ROOT, "include", "dsvg_b200.h")).read()
    body = re.search(r"typedef struct dsvg_epilogue \{(.*?)\} dsvg_epilogue;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = [re.split(r"[\s\*]+", f.strip())[-1] for f in body.split(";") if f.strip()]
    assert names == [f[0] for f in Epilogue._fields_]


def test_outer_problem_struct_matches_header():
    from deepsvg_b200._lib import OuterProblem
    hdr = open(os.path.join(ROOT, "include", "dsvg_b200.h")).read()
    body = re.search(r"typedef struct dsvg_outer_problem \{(.*?)\} dsvg_outer_problem;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for f in body.split(";"):
        f = f.strip()
        if f:
            names += [re.split(r"[\s\*]+", part.strip())[-1] for part in f.split(",")]
    assert names == [f[0] for f in OuterProblem._fields_]


def test_calls_fail_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        return
    from deepsvg_b200 import Hierarchical, SVGTransformer
    import pytest
    model = SVGTransformer(Hierarchical(use_vae=False))
    c = torch.zeros(1, 8, 32)
    a = torch.zeros(1, 8, 32, 11)
    with pytest.raises(RuntimeError, match="no CPU path"):
        model(c, a, c, a)
