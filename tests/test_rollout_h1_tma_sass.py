"""The fp16 form of the persistent rollout kernel (csrc/rollout_fused.cu) stores h1 by TMA, read from the SASS of
csrc/rollout_fused.o (cuobjdump -sass; figures are nvcc 12.9's for sm_90a), for each of its four activations: the
layer-1 epilogue stores h1 with TMA tile stores (UTMASTG) from shared-memory staging, and the stretch from layer 1's last
wgmma wait to the consumers' arrive at cluster barrier 1 holds no per-element global store of h1: at most 8 STG there
(3: the debug trace stamps; the per-element store had 67: two 4-byte stores to the hi / lo planes for each of a thread's
32 accumulator pairs, plus the stamps)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "sample_factory_b200", "csrc", "rollout_fused.o")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

pytestmark = pytest.mark.skipif(not os.path.isfile(OBJ) or not os.path.isfile(CUOBJDUMP),
                                reason="needs csrc/rollout_fused.o (build the library) and cuobjdump")


def _fp16_kernels():
    """{ACT: [opcode with modifiers, ...]} for rollout_mlp2_tape_kernel<ACT, true>"""
    sass = subprocess.run([CUOBJDUMP, "-sass", OBJ], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", line)
        if m and name:
            kernels[name].append(m.group(1))
    out = {}
    for n, ops in kernels.items():
        m = re.match(r"_ZN3sfb24rollout_mlp2_tape_kernelILi(\d)ELb1E", n)
        if m:
            out[int(m.group(1))] = ops
    assert sorted(out) == [0, 1, 2, 3], sorted(out)
    return out


def _layer1_epilogue(ops):
    """the instructions from the last wgmma wait before cluster barrier 1 (the first cluster arrive after the first
    HGMMA) up to that arrive"""
    first_mma = next(i for i, o in enumerate(ops) if o.startswith("HGMMA"))
    arrive = next(i for i, o in enumerate(ops) if o == "UCGABAR_ARV" and i > first_mma)
    wait = max(i for i, o in enumerate(ops[:arrive]) if o.startswith("WARPGROUP.DEPBAR"))
    return ops[wait:arrive]


@pytest.mark.parametrize("act", [0, 1, 2, 3])
def test_h1_is_stored_by_tma(act):
    stretch = _layer1_epilogue(_fp16_kernels()[act])
    assert sum(o.startswith("UTMASTG") for o in stretch) >= 1
    assert sum(o.startswith("STG") for o in stretch) <= 8
