"""CPU: every instantiation of the templated GEMM, attention, LayerNorm, embedding and loss kernels in the built library is
the kernel that at least one case table of tests/test_kernels_gpu.py asserts it launches, or is listed below as
unreachable, with the reason.  A variant that a change makes reachable, or a case that stops reaching its kernel, then
shows up here instead of going untested."""
import os
import re
import shutil
import subprocess

import pytest

import tests.test_kernels_gpu as cases

FAMILIES = re.compile(r"(linear_kernel|outer_kernel|attn_\w+|ln_\w+_kernel|embed_fwd_kernel|ce_args_kernel)\b")

UNREACHABLE = {
    **{"attn_%s_kernel<32, %d%s>" % (k, nt, b): "head_dim 32 with L <= 32 runs the 32 x 32 mma / x3 kernels"
       for nt in (1, 2) for k, b in (("gmma_fwd", ", true"), ("gmma_fwd", ", false"), ("gmma_bwd", ""), ("gx3_fwd", ""),
                                      ("gx3_bwd", ""))},
    **{"attn_gmma_fwd_kernel<%d, %d, false>" % (hd, nt): "launch_gmma stages double-buffered whenever two stages fit in "
       "100 KB, which holds for every <head_dim, tiles> (a compile-time test)" for hd in (32, 64) for nt in range(1, 6)},
}


def _tool(name):
    path = shutil.which(name)
    if path is None and name == "cuobjdump":
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
        path = cand if os.access(cand, os.X_OK) else None
    if path is None:
        pytest.skip("%s not found" % name)
    return path


def _instantiations():
    from deepsvg_b200 import _lib
    _lib.load()
    dump = subprocess.run([_tool("cuobjdump"), "-res-usage", str(_lib.lib_path())], capture_output=True, text=True,
                          check=True).stdout
    mangled = re.findall(r"^\s*Function (\S+):", dump, re.M)
    assert mangled, "cuobjdump listed no kernels"
    names = subprocess.run([_tool("c++filt")], input="\n".join(mangled), capture_output=True, text=True,
                           check=True).stdout.split("\n")
    keys = {cases.kernel_key(n) for n in names if n.strip()}
    return {k for k in keys if k is not None and FAMILIES.match(k)}


def _expected():
    """kernel -> ids of the cases that assert it (the last value of every param in every *_CASES table)."""
    out = {}
    for table in (n for n in dir(cases) if n.endswith("_CASES")):
        for p in getattr(cases, table):
            want = p.values[-1]
            for k in ((want,) if isinstance(want, str) else want):
                out.setdefault(k, []).append("%s[%s]" % (table, p.id))
    return out


def test_every_kernel_instantiation_is_launched_by_a_gpu_case():
    built, expected = _instantiations(), _expected()
    uncovered = sorted(built - set(expected) - set(UNREACHABLE))
    assert not uncovered, "no GPU case asserts a launch of: %s" % ", ".join(uncovered)


def test_case_tables_name_only_compiled_reachable_kernels():
    built, expected = _instantiations(), _expected()
    unknown = sorted(set(expected) - built)
    assert not unknown, "cases expect kernels the library does not contain: %s" % ", ".join(unknown)
    assert not set(UNREACHABLE) - built, sorted(set(UNREACHABLE) - built)
    both = sorted(set(UNREACHABLE) & set(expected))
    assert not both, "listed as unreachable but expected by a case: %s" % both
