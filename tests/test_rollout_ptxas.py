"""The persistent rollout kernel keeps its accumulators in registers: ptxas reports no spill bytes for any instantiation
(the Makefile writes each object's ptxas -v report to csrc/build/<name>.ptxas.log)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "sample_factory_b200", "csrc", "build", "rollout_fused.ptxas.log")


def test_rollout_kernel_has_no_register_spills():
    assert os.path.isfile(LOG), f"{LOG} missing: build the library first (__graft_entry__.build())"
    text = open(LOG).read()
    found = re.findall(r"Function properties for (\S*rollout_mlp2_tape_kernel\S*)\s*\n\s*(\d+) bytes stack frame, "
                       r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(found) == 8, found          # 4 activations x {fp16, tf32} form
    for name, _, stores, loads in found:
        assert int(stores) == 0 and int(loads) == 0, (name, stores, loads)
    assert "rollout_mlp2_tape_kernel" not in "".join(l for l in text.splitlines() if "C7512" in l), \
        "wgmma serialised for lack of registers"
