"""The register epilogues of gemm_wgmma_kernel (csrc/wgmma_tile.cuh) issue their global loads in batches ahead of the
math, read from the SASS of csrc/gemm_tc.o (cuobjdump -sass; figures are nvcc 12.9's for sm_90a).

With one CTA per SM there are two consumer warps per scheduler, so an epilogue that loads, uses and stores pair by pair
pays a load round trip per pair.  Held here, in the code after the kernel's last HGMMA:

* the fp16-form forward <0,0,1,0,1,0> and dX <0,1,1,0,1,0>: somewhere a run of at least 32 LDG with no STG and no BRA
  between them (the whole-tile epilogue loads a thread's 32 bias values, or its 32 float2 of the saved activation, before
  the first store; pair by pair the longest such run is 1);
* the fp16-form forward with the heads folded in <0,0,1,1,1,0>: at most 1000 LDG and 15000 instructions for its four
  activations (744 and 13077: per activation 32 bias loads and eight float2 per (64-column half, head row), shared by
  the thread's two rows; re-loading bias per pair and weights per row took 1570 and 18926)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "sample_factory_b200", "csrc", "gemm_tc.o")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

pytestmark = pytest.mark.skipif(not os.path.isfile(OBJ) or not os.path.isfile(CUOBJDUMP),
                                reason="needs csrc/gemm_tc.o (build the library) and cuobjdump")


def _epilogues():
    """{'<0,1,1,0,1,0>': [opcode, ...] from the last HGMMA on} per gemm_wgmma_kernel instantiation"""
    sass = subprocess.run([CUOBJDUMP, "-sass", OBJ], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_]+)", line)
        if m and name:
            kernels[name].append(m.group(1))
    names = list(kernels)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.splitlines()
    out = {}
    for n, d in zip(names, demangled):
        m = re.match(r"void sfb::gemm_wgmma_kernel<([^>]*)>", d)
        if m:
            key = "<" + ",".join("1" if a.strip() == "true" else "0" for a in m.group(1).split(",")) + ">"
            ops = kernels[n]
            out[key] = ops[max(i for i, o in enumerate(ops) if o == "HGMMA"):]
    return out


def _longest_load_run(ops):
    best = run = 0
    for o in ops:
        if o == "LDG":
            run += 1
            best = max(best, run)
        elif o in ("STG", "BRA"):
            run = 0
    return best


@pytest.mark.parametrize("inst", ["<0,0,1,0,1,0>", "<0,1,1,0,1,0>"])
def test_whole_tile_epilogue_loads_before_it_stores(inst):
    assert _longest_load_run(_epilogues()[inst]) >= 32


def test_heads_epilogue_loads_bias_once_and_weights_once_per_row_pair():
    ops = _epilogues()["<0,0,1,1,1,0>"]
    assert sum(o == "LDG" for o in ops) <= 1000
    assert len(ops) <= 15000
