"""The kernels a CUDA-graph-replayed learner runs between and inside its optimizer steps -- the device learning-rate rules
and the LAMB stages, whose first stage forms the bias corrections from a device step counter -- compile for sm_90a with
no local memory: no stack frame and no spills (the Makefile writes optim.cu's ptxas -v report to
csrc/build/optim.ptxas.log)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "sample_factory_b200", "csrc", "build", "optim.ptxas.log")
KERNELS = {"lr_schedule_kernel", "lamb_stage1_kernel", "lamb_stage2_kernel", "lamb_stage3_kernel"}


def test_schedule_and_lamb_kernels_use_no_local_memory():
    assert os.path.isfile(LOG), f"{LOG} missing: build the library first (__graft_entry__.build())"
    text = open(LOG).read()
    assert "for 'sm_90a'" in text
    found = re.findall(r"Function properties for _ZN3sfb\d+(\w+?_kernel)\w*\s*\n"
                       r"\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    props = {k: (int(a), int(b), int(c)) for k, a, b, c in found if k in KERNELS}
    assert set(props) == KERNELS, props
    for kernel, (stack, stores, loads) in props.items():
        assert stack == 0 and stores == 0 and loads == 0, (kernel, stack, stores, loads)
