"""A forward-only gather over the peer exchange with a local batch SHORTER than the one the exchange was sized for (the
last batch of an eval set): every rank's pooled output equals the unsharded gather of its own rows, bit for bit — with
the kernel model and the tzk_peer.cu source on the host, and with the CUDA kernels on one GPU (W virtual ranks as
threads, tests/test_peer_exchange_model.py's plumbing).  A larger batch is refused before any launch."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import test_peer_exchange_model as M  # noqa: E402
from test_peer_exchange_model import host_compiled_peer_lib  # noqa: E402,F401  (fixture)

from torcheasyrec_b200 import functional as Fn  # noqa: E402
from torcheasyrec_b200 import peer_exchange  # noqa: E402
from torcheasyrec_b200.distributed import TABLE_WISE, _DimGroup, make_plan  # noqa: E402
from torcheasyrec_b200.embedding_modules import EmbeddingBagCollection, output_names_by_table  # noqa: E402

SIZED = 9


def _groups(cfgs, plan, W, full, device):
    names = output_names_by_table(cfgs)
    groups = []
    for r in range(W):
        g = _DimGroup(cfgs, plan, r, W, torch.device(device), True, names)
        g.static_alpha = 2.0
        for t, c in enumerate(cfgs):
            n = g.local._table_rows[t]
            if n:
                start = 0 if plan[c.name].kind == TABLE_WISE else r * plan[c.name].block
                g.local.set_table_weight(t, full.table_weight(t)[start:start + n])
        groups.append(g)
    return groups


def _short_gather(backend, device, W, sizes, multi_hot):
    rng = np.random.default_rng(W * 7 + sum(sizes))
    cfgs = M._pooled_configs()
    plan = make_plan(cfgs, W, "row_wise", {"t_tw": [TABLE_WISE]})
    with Fn.use_backend(backend):
        full = EmbeddingBagCollection(cfgs, device=device)
        F = len(full.feature_names())
        feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
        groups = _groups(cfgs, plan, W, full, device)
        batches = [[t.to(device) for t in M._bags(rng, F, b, feat_rows, multi_hot)] for b in sizes]
        registry, outs = {}, [None] * W

        def body(r, tbar):
            if device != "cpu":
                torch.cuda.set_device(0)

            class St(M._sim_mixin(registry, tbar, f"short{W}", device), peer_exchange.PeerState):
                pass

            st = St(groups[r], plan, None, SIZED, [SIZED * 4] * F)
            with torch.no_grad():
                outs[r] = st.gather(*batches[r], B=sizes[r])
            if device != "cpu":
                torch.cuda.synchronize()
            with pytest.raises(RuntimeError, match="sized for local batches"):
                st.gather(*batches[r], B=SIZED + 1)

        M._run_ranks(W, body)
        for r in range(W):
            want = backend.pooled_gather_fwd(full.weights.data, full.layout, batches[r][0], batches[r][1], sizes[r])
            assert outs[r].shape == (sizes[r], full.layout.total_dim)
            assert torch.equal(outs[r].cpu(), want.cpu()), r


@pytest.mark.parametrize("kernels", ["model", "source"])
@pytest.mark.parametrize("W,sizes,multi_hot", [(2, (4, 9), True), (3, (1, 5, 8), False), (2, (3, 3), True)])
def test_short_batch_gather_equals_unsharded(kernels, W, sizes, multi_hot, host_compiled_peer_lib):  # noqa: F811
    backend = M.OracleKernels() if kernels == "model" else M.SourceKernels(host_compiled_peer_lib)
    _short_gather(backend, "cpu", W, sizes, multi_hot)


@pytest.mark.gpu
@pytest.mark.parametrize("W,sizes,multi_hot", [(2, (4, 9), True), (3, (1, 5, 8), False)])
def test_short_batch_gather_on_one_gpu(kernels, W, sizes, multi_hot):
    _short_gather(kernels, "cuda", W, sizes, multi_hot)
