"""The head partials of the fp16-form heads GEMM (gemm_wgmma_kernel<0,0,1,1,1,0>) and of the fp16-form persistent rollout
(rollout_mlp2_tape_kernel<ACT, true>) run on the tensor cores (head_partials_f16 in csrc/wgmma_tile.cuh), read from the
SASS of csrc/gemm_tc.o and csrc/rollout_fused.o (cuobjdump -sass; figures are nvcc 12.9's for sm_90a):

* the heads GEMM issues them as the engine's register-A `HGMMA.64x128x16.F32 Rd, Ra, gdesc[..].tnspB` with B MN-major
  (16 per activation: two 64-column halves x two passes x four k16 steps), which no mainloop HGMMA of the fp16 forward
  uses;
* after its last mainloop HGMMA there are fewer FFMA than the FMA partials of its four activations took alone
  (4 x 576 per thread, 36 dependent chains of 16 each; 3270 FFMA in all with them);
* the fp16-form rollout kernels issue the same 16 as `HGMMA.64x64x16.F32 Rd, Ra, gdesc[..].tnspB`, the tf32-form ones
  none."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "sample_factory_b200", "csrc")
GEMM_OBJ = os.path.join(CSRC, "gemm_tc.o")
ROLLOUT_OBJ = os.path.join(CSRC, "rollout_fused.o")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

pytestmark = pytest.mark.skipif(not all(os.path.isfile(p) for p in (GEMM_OBJ, ROLLOUT_OBJ, CUOBJDUMP)),
                                reason="needs csrc/gemm_tc.o, csrc/rollout_fused.o (build the library) and cuobjdump")

HEADS = "<0,0,1,1,1,0>"
PART_RE = r"HGMMA\.64x128x16\.F32 R\d+, R\d+, gdesc\[[^\]]*\]\.tnspB"
ROLLOUT_PART_RE = r"HGMMA\.64x64x16\.F32 R\d+, R\d+, gdesc\[[^\]]*\]\.tnspB"


def _sass(obj):
    """{demangled kernel name: [instruction text, ...]}"""
    sass = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
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
    return {d: kernels[n] for n, d in zip(names, demangled)}


def _flags(args):
    return "<" + ",".join("1" if a.strip() == "true" else "0" for a in args.split(",")) + ">"


@pytest.fixture(scope="module")
def gemm():
    out = {}
    for d, ins in _sass(GEMM_OBJ).items():
        m = re.match(r"void sfb::gemm_wgmma_kernel<([^>]*)>", d)
        if m:
            out[_flags(m.group(1))] = ins
        elif d.startswith("sfb::gemm_dw_f16_kernel"):
            out["dw16"] = ins
    return out


@pytest.fixture(scope="module")
def rollout():
    out = {}
    for d, ins in _sass(ROLLOUT_OBJ).items():
        m = re.match(r"void sfb::rollout_mlp2_tape_kernel<(-?\d+), (true|false)>", d)
        if m:
            out[(int(m.group(1)), m.group(2) == "true")] = ins
    return out


def test_heads_gemm_partials_on_tensor_cores(gemm):
    ins = gemm[HEADS]
    assert sum(bool(re.match(PART_RE, i)) for i in ins) == 4 * 16   # four activations
    assert not any(re.match(PART_RE, i) for i in gemm["<0,0,1,0,1,0>"])
    last_main = max(j for j, i in enumerate(ins) if i.startswith("HGMMA") and not re.match(PART_RE, i))
    ffma = sum(i.split()[0].startswith("FFMA") for i in ins[last_main:])
    assert ffma < 4 * 576, ffma


def test_rollout_partials_on_tensor_cores(rollout):
    assert len(rollout) == 8, sorted(rollout)
    for (act, f16), ins in rollout.items():
        n = sum(bool(re.match(ROLLOUT_PART_RE, i)) for i in ins)
        assert n == (16 if f16 else 0), (act, f16, n)
