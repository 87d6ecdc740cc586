"""How sensitive are the tables of the BASELINE models, after two fused Adagrad steps, to ulp-level noise in the dense path?

`verify_sharded` (torcheasyrec_b200/verify.py, the in-bench `verify`) compares the sharded step's tables with an unsharded
twin at rtol 5e-5 / atol 1e-6.  The twin runs its dense towers on the concatenated batch (W x B rows), the ranks on B rows:
GEMM tilings differ, so the per-sample gradients differ by a few ulp.  Adagrad's first steps divide by sqrt(sum g^2) + 1e-8:
gradient elements of the order of eps are amplified to O(lr).  This script steps two CPU twins (oracle backend) on the same
2048-sample batch, the second with every dense parameter scaled by (1 + 1e-7 N(0,1)), and counts the table elements that
the verify tolerance would flag:

    mmoe_taobao             7625 violations, worst 5.6e-4
    multi_tower_din_taobao    81 violations, worst 2.0e-4
    dlrm_criteo                0 violations, worst 1.2e-7

i.e. a small MMoE `verify` deviation at N>1 can be inside what one-ulp noise does to this model; it is not evidence of
a plumbing error (the same tables and plan pass with DIN's gradients), and not proof of its absence either.
    python scripts/verify_sensitivity.py
"""
import sys, numpy as np, torch
import os; ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle_backend import OracleKernels
from torcheasyrec_b200 import functional as Fn
from torcheasyrec_b200.engine import Pipeline
from torcheasyrec_b200.verify import concat_batches
torch.set_num_threads(8)
def run(name, scale_noise):
    a=Pipeline(name, device="cpu", max_rows=2000, seed=5)
    b=Pipeline(name, device="cpu", max_rows=2000, seed=5)
    b.model.load_state_dict(a.model.state_dict())
    batches=[a.synthetic_batch(256, seed=77+r) for r in range(8)]
    glob=concat_batches(batches)
    # twin b: dense parameters perturbed by 1 ulp-level relative noise (emulates a different GEMM summation order)
    g=torch.Generator().manual_seed(0)
    with torch.no_grad():
        for p in b.model.dense_parameters():
            p.mul_(1.0 + scale_noise*torch.randn(p.shape, generator=g))
    with Fn.use_backend(OracleKernels()):
        for _ in range(2):
            a.eager_step(glob); b.eager_step(glob)
    worst=0; cnt=0
    for ca,cb in zip(a.model.sparse_collections(), b.model.sparse_collections()):
        for t,c in enumerate(ca._configs):
            x=ca.table_weight(t).numpy(); y=cb.table_weight(t).numpy()
            bad=np.abs(x-y) > (1e-6+5e-5*np.abs(y))
            if bad.any(): print(name, c.name, "violations", int(bad.sum()), "max abs", float(np.abs(x-y)[bad].max()))
            worst=max(worst, float(np.abs(x-y).max())); cnt+=int(bad.sum())
    print(name, "noise", scale_noise, "worst abs dev", worst, "violations", cnt)
for name in ("mmoe_taobao","multi_tower_din_taobao","dlrm_criteo"):
    run(name, 1e-7)
