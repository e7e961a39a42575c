"""The C-ABI library loads and exports every symbol include/bioik_b200.h declares (no compute calls: CPU)."""
import ctypes as C
import os
import re

import pytest

import __graft_entry__ as ge
from bio_ik_b200 import _abi


@pytest.fixture(scope="module")
def lib():
    ge.build_cuda()
    return C.CDLL(_abi.LIB_PATH)


def test_exports_every_declared_symbol(lib):
    hdr = open(os.path.join(_abi.REPO_ROOT, "include", "bioik_b200.h")).read()
    declared = set(re.findall(r"\b(bioik_[a-z_]+)\s*\(", hdr))
    assert declared == set(_abi.ABI_SYMBOLS), declared ^ set(_abi.ABI_SYMBOLS)
    for sym in declared:
        assert hasattr(lib, sym), sym


def test_abi_version_and_struct_sizes(lib):
    lib.bioik_abi_version.restype = C.c_int
    assert lib.bioik_abi_version() == 2
    # POD layout agreed with the header (LP64)
    assert C.sizeof(_abi.BioikGoal) == 16 + 8 + 8 * _abi.GOAL_NPARAM
    assert C.sizeof(_abi.BioikSolverCfg) == 24
    assert C.sizeof(_abi.BioikRobot) == 8 + 14 * 8
    assert C.sizeof(_abi.BioikProblem) == 3 * 16 + 3 * 8


def test_sm90a_code_and_no_oracle_linkage(lib):
    """The shipped library carries sm_90a SASS and does not link or reference the oracle."""
    import subprocess
    out = subprocess.run(["cuobjdump", "--list-elf", _abi.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    ldd = subprocess.run(["ldd", _abi.LIB_PATH], capture_output=True, text=True).stdout
    assert "oracle" not in ldd and "hostsim" not in ldd
    syms = subprocess.run(["nm", "-D", _abi.LIB_PATH], capture_output=True, text=True).stdout
    assert "oracle_" not in syms and "hostsim_" not in syms


def test_python_binding_prototypes():
    lib = _abi.load_library()
    for sym in _abi.ABI_SYMBOLS:
        assert getattr(lib, sym).restype is not None or sym == "bioik_destroy"
