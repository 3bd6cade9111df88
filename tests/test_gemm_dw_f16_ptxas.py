"""gemm_dw_f16_kernel (the fp16 form of dW, csrc/gemm_tc.cu) keeps its two 64-register accumulators in registers like the
other GEMM instantiations: no spills, and no more than the 168 registers per thread a 384-thread, one-CTA-per-SM launch
gets (read from csrc/build/gemm_tc.ptxas.log, which the Makefile writes; figures are nvcc 12.9's for sm_90a)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "sample_factory_b200", "csrc", "build", "gemm_tc.ptxas.log")


def test_dw_f16_kernel_fits_without_spills():
    assert os.path.isfile(LOG), f"{LOG} missing: build the library first (__graft_entry__.build())"
    found = re.findall(r"Function properties for (\S*gemm_dw_f16_kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes "
                       r"spill stores, (\d+) bytes spill loads\s*\n(?:ptxas info\s*: Compiling.*\n)?ptxas info\s*: Used "
                       r"(\d+) registers", open(LOG).read())
    assert len(found) == 1, found
    _, frame, stores, loads, regs = found[0]
    assert int(frame) == 0 and int(stores) == 0 and int(loads) == 0, found[0]
    assert int(regs) <= 168, found[0]
