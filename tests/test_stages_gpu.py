"""Per-stage parity (SURVEY section 8 rows a3-a18 one by one): the evaluation is run one launch at a time
(``vb_debug_run``) and every buffer a stage produces is compared with the fp64 hand-adjoint oracle
(``oracle/adjoint_ref.py``, equal to autograd at 1e-14).  Covered: the default plan (SIMT node stage, both edge stages
on tensor cores), every other combination of SIMT and tensor-core edge stages ("edge_tc" 0, 1, 2), the tensor-core node
stage and the SIMT node kernels of NB = 1, 2, 3, 4 and 8 nodes per CTA, all on the first four Chignolin fragments (one
edge tile per CTA).  NB = 16 ("npw" 2), several tiles per CTA and the production-size variants are in
test_kernel_variants_gpu.py.
Tolerance: 2e-3 relative to the largest reference entry of the buffer (fp32 + 3xTF32 against fp64; measured
1e-6 .. 3e-4, adjoint buffers deep in the reverse sweep being the largest)."""
import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tools"))

pytestmark = pytest.mark.gpu


# default here: node_nb=1 (one wave); test_stale_workspace_gpu.py runs the same list after a decoy geometry
OPTS = ["", "edge_tc=0", "edge_tc=1", "edge_tc=2", "node_tc=1", "node_nb=2", "node_nb=3", "node_nb=4", "node_nb=8"]


@pytest.mark.parametrize("opts", OPTS, ids=lambda o: o or "default")
@pytest.mark.parametrize("weights", ["real", "3"])
def test_every_stage_against_the_fp64_adjoint_oracle(opts, weights):
    from stage_check import stage_report
    lines, worst = stage_report("chig", weights, max_frags=4, opts=opts)
    bad = [(s, w, r) for s, w, r in worst if not r <= 2e-3]
    assert not bad, "\n".join(lines)
    stages = {s for s, _, _ in worst}
    assert "head" in stages and "embed_node_bwd" in stages and "finalize" in stages
    assert ("proj3" in stages and "bwdB2" in stages) == ("node_tc=1" in opts)
