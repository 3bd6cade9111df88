"""The fp16-form mainloops of the wgmma GEMM (csrc/gemm_tc.cu) take the A operand from registers and keep two groups of
wgmmas in flight, read from the SASS of csrc/gemm_tc.o (cuobjdump -sass; figures are nvcc 12.9's for sm_90a):

* in the fp16 forward <0,0,1,0,1,0>, dX <0,1,1,0,1,0>, forward with the heads <0,0,1,1,1,0> and gemm_dw_f16_kernel,
  every HGMMA reads A from registers (`HGMMA.64x128x16.F32 Rd, Ra, gdesc[..]`), none from a shared-memory descriptor;
* they wait with `WARPGROUP.DEPBAR.LE gsb0, 0x1` (wgmma.wait_group 1: the group just issued stays in flight);
* the three gemm_wgmma_kernel instantiations have no BAR.SYNC between their first and last HGMMA: the consumer
  warpgroups meet only at mbarriers in the mainloop."""
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

F16_FORMS = ["<0,0,1,0,1,0>", "<0,1,1,0,1,0>", "<0,0,1,1,1,0>"]


def _kernels():
    """{'<0,1,1,0,1,0>' or 'dw16': [instruction text, ...]} for the fp16-form GEMM kernels"""
    sass = subprocess.run([CUOBJDUMP, "-sass", OBJ], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([^;]*);", line)
        if m and name:
            kernels[name].append(m.group(1).strip())
    names = list(kernels)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True,
                               check=True).stdout.splitlines()
    out = {}
    for n, d in zip(names, demangled):
        m = re.match(r"void sfb::gemm_wgmma_kernel<([^>]*)>", d)
        if m:
            out["<" + ",".join("1" if a.strip() == "true" else "0" for a in m.group(1).split(",")) + ">"] = kernels[n]
        elif d.startswith("sfb::gemm_dw_f16_kernel"):
            out["dw16"] = kernels[n]
    return out


@pytest.fixture(scope="module")
def kernels():
    return _kernels()


@pytest.mark.parametrize("inst", F16_FORMS + ["dw16"])
def test_hgmma_takes_a_from_registers(kernels, inst):
    hgmma = [i for i in kernels[inst] if i.startswith("HGMMA")]
    assert len(hgmma) >= 6, hgmma
    for i in hgmma:
        assert re.match(r"HGMMA\.64x128x16\.F32 R\d+, R\d+, gdesc\[", i), i


@pytest.mark.parametrize("inst", F16_FORMS + ["dw16"])
def test_mainloop_keeps_one_group_in_flight(kernels, inst):
    assert any(re.match(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", i) for i in kernels[inst])


@pytest.mark.parametrize("inst", F16_FORMS)
def test_no_barrier_between_hgmmas(kernels, inst):
    ops = [i.split()[0] for i in kernels[inst]]
    first = ops.index(next(o for o in ops if o.startswith("HGMMA")))
    last = max(j for j, o in enumerate(ops) if o.startswith("HGMMA"))
    assert not [o for o in ops[first:last] if o.startswith("BAR.SYNC")]
