"""Register spills of the loss and action-ratio kernels do not grow (the Makefile writes each object's ptxas -v report to
csrc/build/<name>.ptxas.log): no one-thread-per-sample instantiation and no ratio kernel spills, no one-warp-per-sample
loss instantiation spills more than the figures below (nvcc 12.9, sm_90a), and the plain-Discrete loss of the bench
workload (A <= 8) keeps to 67 registers."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "sample_factory_b200", "csrc", "build", "loss.ptxas.log")

# (kernel, elements per lane) -> (spill store, spill load) bytes allowed; warp-per-sample loss kernels not listed: none
WIDE_LOSS_SPILLS = {
    ("ppo_loss_wide_kernel", 2): (12, 12), ("ppo_loss_wide_kernel", 32): (120, 120),
    ("ppo_loss_tuple_wide_kernel", 32): (192, 272),
    ("ppo_loss_gauss_wide_kernel", 32): (4, 4),
    ("ppo_loss_mixed_kernel", 2): (28, 28), ("ppo_loss_mixed_kernel", 16): (280, 356),
    ("ppo_loss_mixed_kernel", 32): (88, 120),
}
THREAD_PER_SAMPLE = {"ppo_loss_kernel", "ppo_loss_tuple_kernel", "ppo_loss_gauss_kernel"}


def _kernels():
    assert os.path.isfile(LOG), f"{LOG} missing: build the library first (__graft_entry__.build())"
    text = open(LOG).read()
    found = re.findall(r"Function properties for _ZN3sfb\d+((?:ppo_loss|action_ratio)\w*?_kernel)ILi(\d+)EE\w*\s*\n"
                       r"\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\s*\n"
                       r"ptxas info\s*: Used (\d+) registers", text)
    return [(k, int(n), int(st), int(ld), int(regs)) for k, n, st, ld, regs in found]


def test_loss_kernels_spill_no_more_than_listed():
    found = _kernels()
    # 3 thread-per-sample loss + 3 ratio kernels x 3 widths, 3 wide loss + 2 wide ratio kernels x 5 widths,
    # the mixed loss and ratio kernels x 6 widths
    assert len(found) == 6 * 3 + 5 * 5 + 2 * 6, found
    for kernel, n, stores, loads, _ in found:
        if kernel.startswith("action_ratio") or kernel in THREAD_PER_SAMPLE:
            assert stores == 0 and loads == 0, (kernel, n, stores, loads)
        else:
            st_max, ld_max = WIDE_LOSS_SPILLS.get((kernel, n), (0, 0))
            assert stores <= st_max and loads <= ld_max, (kernel, n, stores, loads)


def test_bench_loss_kernel_registers():
    # registers only: that this instantiation does not spill is asserted above, with every thread-per-sample kernel
    regs = [r for k, n, _, _, r in _kernels() if (k, n) == ("ppo_loss_kernel", 8)]
    assert len(regs) == 1 and regs[0] <= 67, regs
