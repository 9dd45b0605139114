"""CPU tier: every kernel launched with IM_LAUNCH_PDL waits for its predecessor (griddepcontrol.wait in its sm_90a PTX).  A kernel
launched with the programmatic attribute that never waits would let its own successor start before its predecessor has finished."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "immesh_b200", "csrc")


def pdl_kernels(src):
    """names of the kernels at the IM_LAUNCH_PDL sites of `src` (second macro argument)"""
    txt = open(os.path.join(CSRC, src)).read()
    return sorted(set(re.findall(r"IM_LAUNCH_PDL\([^,]+,\s*\(?([A-Za-z_]\w*)", txt)) - {"KERN"})


def ptx_entries(src, out_dir):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    ptx = os.path.join(out_dir, src + ".ptx")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-ptx", "-w", "-o", ptx, os.path.join(CSRC, src)],
                   check=True, capture_output=True)
    txt = open(ptx).read()
    entries = {}
    for m in re.finditer(r"\.entry\s+(\S+)\(", txt):
        end = txt.find("\n}\n", m.end())
        entries[m.group(1)] = txt[m.end():end]
    return entries


@pytest.mark.parametrize("src,n_min", [("lio_capi.cu", 10), ("mesh_capi.cu", 14)])
def test_pdl_kernels_wait(src, n_min):
    names = pdl_kernels(src)
    assert len(names) >= n_min, names
    with tempfile.TemporaryDirectory() as td:
        entries = ptx_entries(src, td)
    for name in names:
        mangled = f"_Z{len(name)}{name}"
        bodies = [b for e, b in entries.items() if e.startswith(mangled)]
        assert bodies, f"{name}: no PTX entry"
        for b in bodies:
            assert "griddepcontrol.wait" in b, f"{name} is launched with IM_LAUNCH_PDL but never waits for its predecessor"
