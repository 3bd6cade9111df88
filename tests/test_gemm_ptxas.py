"""gemm_wgmma_kernel (csrc/gemm_tc.cu) keeps its accumulators in registers: every instantiation compiles without a byte
of spills (the Makefile writes ptxas -v's report to csrc/build/gemm_tc.ptxas.log; figures are nvcc 12.9's for sm_90a).
The kernel is launched with 384 threads, one CTA per SM, so 168 registers per thread is all a launch gets; the item loop
of the persistent kernel lives beside two 64-register accumulators only because the producer warpgroup hands registers
over (setmaxnreg), which the report does not show -- spills it would."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "sample_factory_b200", "csrc", "build", "gemm_tc.ptxas.log")

# <A_MN, B_MN, SPLIT3, HEADS, F16, RES>: four operand layouts x {1-pass, 3-pass} tf32, HEADS and RES in both, and the
# fp16 form's forward, dX and HEADS
INSTANTIATIONS = 15


def _kernels():
    assert os.path.isfile(LOG), f"{LOG} missing: build the library first (__graft_entry__.build())"
    found = re.findall(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads\s*\n(?:ptxas info\s*: Compiling.*\n)?ptxas info\s*: Used (\d+) registers",
                       open(LOG).read())
    names = subprocess.run(["c++filt"], input="\n".join(f[0] for f in found), capture_output=True, text=True,
                           check=True).stdout.splitlines()
    return [(re.sub(r"\(.*", "", n), int(fr), int(st), int(ld), int(r)) for n, (_, fr, st, ld, r) in zip(names, found)
            if "gemm_wgmma_kernel" in n]


def test_no_instantiation_spills():
    kernels = _kernels()
    assert len(kernels) == INSTANTIATIONS, [k[0] for k in kernels]
    for name, frame, stores, loads, regs in kernels:
        assert frame == 0 and stores == 0 and loads == 0, (name, frame, stores, loads)
        assert regs <= 168, (name, regs)


def test_heads_instantiations_fit_the_launch():
    heads = [k for k in _kernels() if re.match(r"void sfb::gemm_wgmma_kernel<\w+, \w+, \w+, true,", k[0])]
    assert len(heads) == 3, heads
    for name, frame, stores, loads, regs in heads:
        assert stores == 0 and loads == 0 and regs <= 168, (name, stores, loads, regs)
