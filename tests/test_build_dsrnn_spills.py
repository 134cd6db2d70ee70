"""Static check of the built library (cuobjdump needs no GPU): the DS-RNN forward's kernels keep everything in registers.
A spill to local memory in the edge-GRU GEMM (128 accumulator registers per thread plus the gate math of its epilogue)
or in the per-row kernels would put it on the HBM path of every rollout step."""
import os
import re
import shutil
import subprocess

import pytest

from crowdnav_prediction_attngraph_b200 import _capi

# mangled-name fragments: the TC_OUT_GRU instance of cn_gemm_tc_kernel, the dense robot-human attention, the two
# DS-RNN input kernels
KERNELS = ["cn_gemm_tc_kernelILi256ELb0ELi0ELi4E", "cn_hr_attention_kernelILb1E", "cn_dsrnn_edge_pack_kernel",
           "cn_dsrnn_node_in_kernel"]


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_dsrnn_kernels_use_no_local_memory():
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    out = subprocess.run(["cuobjdump", "-res-usage", _capi.LIB_PATH], capture_output=True, text=True).stdout
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out))
    for frag in KERNELS:
        hits = {name: u for name, u in usage.items() if frag in name}
        assert hits, "kernel %s not in the library" % frag
        for name, u in hits.items():
            assert re.search(r"\bSTACK:0\b", u) and re.search(r"\bLOCAL:0\b", u), (name, u)
