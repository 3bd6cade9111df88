"""Register spills of the heads kernels do not grow (the Makefile writes each object's ptxas -v report to
csrc/build/<name>.ptxas.log); the figures are nvcc 12.9's for sm_90a.  The GEMMs that finish the heads in their epilogue (HEADS = true) sit at the
384-thread register cap, so they must stay at 168 registers or fewer without spilling; heads_from_partials_kernel,
which runs on the learner's path, keeps to 48 registers, and sampler_tail_tape_kernel to 128."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "sample_factory_b200", "csrc", "build")

# demangled kernel -> (spill store, spill load) bytes allowed; kernels not listed: none
SPILLS = {
    "void sfb::heads_forward_kernel<32, 1, true>": (20, 12),
}
NARROW = {"heads_forward_kernel": 7, "heads_from_partials_kernel": 1, "sampler_tail_tape_kernel": 1}


def _kernels(log):
    path = os.path.join(BUILD, log)
    assert os.path.isfile(path), f"{path} missing: build the library first (__graft_entry__.build())"
    found = re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads\s*\n(?:ptxas info\s*: Compiling.*\n)?ptxas info\s*: Used (\d+) registers",
                       open(path).read())
    names = subprocess.run(["c++filt"], input="\n".join(f[0] for f in found), capture_output=True, text=True,
                           check=True).stdout.splitlines()
    return [(re.sub(r"\(.*", "", n), int(st), int(ld), int(r)) for n, (_, st, ld, r) in zip(names, found)]


def _check(kernels):
    for name, stores, loads, _ in kernels:
        st_max, ld_max = SPILLS.get(name, (0, 0))
        assert stores <= st_max and loads <= ld_max, (name, stores, loads)


def test_narrow_heads_kernels_spill_no_more_than_listed():
    found = [k for k in _kernels("heads.ptxas.log") if any(n in k[0] for n in NARROW)]
    for n, count in NARROW.items():
        assert sum(n in k[0] for k in found) == count, (n, found)
    _check(found)
    regs = [r for name, _, _, r in found if name == "sfb::heads_from_partials_kernel"]
    assert regs[0] <= 48, regs
    regs = [r for name, _, _, r in found if name == "sfb::sampler_tail_tape_kernel"]
    assert regs[0] <= 128, regs


def test_stored_row_tail_does_not_spill():
    found = [k for k in _kernels("heads_wide.ptxas.log") if "heads_tail_rows_kernel" in k[0]]
    assert len(found) == 11, found        # LPL 1..32 with S = 0 (mixed Tuple), LPL 2..32 with S = 1 (wide heads)
    _check(found)


def test_gemm_heads_epilogue_registers():
    # gemm_wgmma_kernel<A_MN, B_MN, SPLIT3, HEADS, ...>: the instantiations that finish the heads
    found = [k for k in _kernels("gemm_tc.ptxas.log")
             if re.match(r"void sfb::gemm_wgmma_kernel<\w+, \w+, \w+, true,", k[0])]
    assert len(found) == 3, found
    for name, stores, loads, regs in found:
        assert stores == 0 and loads == 0 and regs <= 168, (name, stores, loads, regs)
