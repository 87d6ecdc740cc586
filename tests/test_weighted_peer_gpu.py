"""Weighted id features on the peer-memory sparse step, on ONE GPU: W virtual ranks are threads of this process whose
"symmetric" buffers are allocations of the same device (tests/test_peer_gpu.py's setup) — the CUDA kernels through the
C-ABI, `PeerState`, side streams.  Checked against the unsharded weighted CUDA collection:
  * step 0: every rank's forward has the bits of pooled_gather_fwd(per_sample_weights=...), one-launch and split gather;
  * tables after two steps within 5e-5 of the unsharded weighted fused_bwd on the concatenated batch (grad / W), for
    Adagrad, row-wise Adagrad, Adam and LAMB (the norm family);
  * SGD with lr = -1 on a zero arena with dyadic data: every touched row is its float64 gradient sum, bit for bit
    (a hot row with long runs, mirrored tables);
  * all-ones weights: the unweighted peer step bit for bit.
Two real GPUs: the Ali-CCP MMoE config (nine weighted features) sharded over peer memory against its unsharded twin."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

pytestmark = pytest.mark.gpu
f32 = np.float32


def _helpers():
    import test_peer_exchange_model as M
    import test_peer_gpu as G

    return M, G


def _bags(rng, F, B, feat_rows, lens_from=(0, 1, 2, 3, 4), hot=None):
    """Ragged multi-hot bags (empty ones included); hot = (feature, row, p): that share of feature f's ids is `row`."""
    lens = rng.choice(list(lens_from), F * B)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    parts = []
    for b in range(F * B):
        ids = rng.integers(0, feat_rows[b // B], lens[b])
        if hot is not None and b // B == hot[0]:
            ids = np.where(rng.random(lens[b]) < hot[2], hot[1], ids)
        parts.append(ids)
    ids = np.concatenate(parts + [np.zeros(0, np.int64)]).astype(np.int64)
    return torch.from_numpy(ids).cuda(), torch.from_numpy(off).cuda()


def _run(W, B, spec, full, cfgs, plan, batches, weights, grads, tag, steps=2, budget_per_bag=4):
    M, G = _helpers()
    from torcheasyrec_b200 import peer_exchange

    F = len(full.feature_names())
    groups = G._seed_groups(cfgs, plan, W, True, full, spec, 2.5)
    registry, outs = {}, [[None] * W for _ in range(steps)]

    def body(r, tbar):
        torch.cuda.set_device(0)

        class St(M._sim_mixin(registry, tbar, tag, "cuda"), peer_exchange.PeerState):
            pass

        st = St(groups[r], plan, None, B, [B * budget_per_bag] * F)
        psw = None if weights is None else weights[r]
        for s in range(steps):
            outs[s][r] = st.gather(batches[r][0], batches[r][1], psw).clone()
            if grads is None:
                torch.cuda.synchronize()
                continue
            st.prep(batches[r][0], batches[r][1], psw)
            st.backward(grads[r], batches[r][1])
            torch.cuda.synchronize()

    M._run_ranks(W, body)
    assert all(int(g.overflow.item()) == 0 for g in groups)
    return groups, outs


def _concat(M, batches, weights, F, B, W):
    ids = [b[0].cpu() for b in batches]
    offs = [b[1].cpu() for b in batches]
    cat_ids, cat_off = M._cat_key_major(ids, offs, F, B, W)
    cat_w = torch.cat([weights[r].cpu()[offs[r][f * B]:offs[r][(f + 1) * B]] for f in range(F) for r in range(W)])
    return cat_ids.cuda(), cat_off.cuda(), cat_w.cuda()


def _setup(W, opt, seed, lr=0.05):
    M, _ = _helpers()
    from torcheasyrec_b200.distributed import TABLE_WISE, make_plan
    from torcheasyrec_b200.embedding_modules import EmbeddingBagCollection, SparseOptimizerSpec

    torch.manual_seed(seed)
    cfgs = M._pooled_configs()       # SUM / MEAN, a shared table, a 2-row table, a table-wise one; small ones mirrored
    plan = make_plan(cfgs, W, "row_wise", {"t_tw": [TABLE_WISE], "t_tiny": [TABLE_WISE]})
    spec = SparseOptimizerSpec.from_name(opt, lr=lr)
    full = EmbeddingBagCollection(cfgs, device="cuda")
    full.set_optimizer(spec)
    return M, cfgs, plan, spec, full


@pytest.mark.parametrize("split", ["0", "1"])
@pytest.mark.parametrize("B", [64, 257, 4099])
def test_weighted_peer_forward_is_the_unsharded_weighted_gather(kernels, monkeypatch, B, split):
    monkeypatch.setenv("TZK_PEER_SPLIT_GATHER", split)
    W = 3
    M, cfgs, plan, spec, full = _setup(W, "adagrad", 1)
    rng = np.random.default_rng(B + int(split))
    F = len(full.feature_names())
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    batches = [_bags(rng, F, B, feat_rows) for _ in range(W)]
    weights = [torch.from_numpy(rng.standard_normal(b[0].numel()).astype(f32)).cuda() for b in batches]
    _, outs = _run(W, B, spec, full, cfgs, plan, batches, weights, None, "fwd" + split, steps=1)
    for r in range(W):
        want = kernels.pooled_gather_fwd(full.weights.data, full.layout, batches[r][0], batches[r][1], B,
                                         per_sample_weights=weights[r])
        assert torch.equal(outs[0][r], want), r


@pytest.mark.parametrize("opt", ["adagrad", "rowwise_adagrad", "adam", "lamb"])
def test_weighted_peer_tables_match_unsharded(kernels, opt):
    W, B = 4, 1000
    M, cfgs, plan, spec, full = _setup(W, opt, 2)
    rng = np.random.default_rng(17)
    F = len(full.feature_names())
    D = 16
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    batches = [_bags(rng, F, B, feat_rows) for _ in range(W)]
    weights = [torch.from_numpy((rng.standard_normal(b[0].numel()) * 1.5).astype(f32)).cuda() for b in batches]
    grads = [torch.from_numpy(rng.standard_normal((B, F * D)).astype(f32)).cuda() for _ in range(W)]
    groups, outs = _run(W, B, spec, full, cfgs, plan, batches, weights, grads, "tab" + opt)
    cat_ids, cat_off, cat_w = _concat(M, batches, weights, F, B, W)
    cat_grad = torch.cat(grads) / W
    for step in range(2):
        for r in range(W):
            want = kernels.pooled_gather_fwd(full.weights.data, full.layout, batches[r][0], batches[r][1], B,
                                             per_sample_weights=weights[r])
            if step == 0:
                assert torch.equal(outs[0][r], want)
            else:
                torch.testing.assert_close(outs[1][r], want, rtol=2e-5, atol=1e-6)
        kernels.fused_bwd(spec.kind, True, cat_grad, full.weights.data, full.opt_state, full.layout, cat_ids, cat_off,
                          B * W, spec.lr, spec.eps, 1.0, per_sample_weights=cat_w, **full.opt_extras())
    _, G = _helpers()
    for t, c in enumerate(cfgs):
        torch.testing.assert_close(G._gathered(groups, plan, cfgs, full, t), full.table_weight(t), rtol=5e-5, atol=1e-6,
                                   msg=lambda m, c=c: f"{c.name}: {m}")


@pytest.mark.parametrize("W", [2, 4])
def test_weighted_peer_exact_row_sums(kernels, W):
    """SGD, lr = -1, zero arena: a touched row ends as sum_l w[l] * g_bag (/ L) / W over every rank's ids.  Dyadic data
    (weights k/4, gradients k/8, bag lengths 1, 2 or 4, W a power of two) makes every product and sum exact in fp32,
    so each row must equal its float64 sum bit for bit — whatever order the sharded and the mirrored paths add in."""
    B = 4099
    M, cfgs, plan, spec, full = _setup(W, "sgd", 3, lr=-1.0)
    full.weights.data.zero_()
    rng = np.random.default_rng(29 + W)
    F = len(full.feature_names())
    D = 16
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    batches = [_bags(rng, F, B, feat_rows, lens_from=(0, 1, 2, 4), hot=(0, 5, 0.3)) for _ in range(W)]
    weights = [torch.from_numpy((rng.integers(-8, 9, b[0].numel()) / 4.0).astype(f32)).cuda() for b in batches]
    grads = [torch.from_numpy((rng.integers(-8, 9, (B, F * D)) / 8.0).astype(f32)).cuda() for _ in range(W)]
    groups, _ = _run(W, B, spec, full, cfgs, plan, batches, weights, grads, f"exact{W}", steps=1)
    lay = full.layout
    want = [np.zeros((c.num_embeddings, c.embedding_dim), np.float64) for c in cfgs]
    touched = [np.zeros(c.num_embeddings, bool) for c in cfgs]
    for r in range(W):
        ids, off = batches[r][0].cpu().numpy(), batches[r][1].cpu().numpy()
        w, g = weights[r].cpu().numpy().astype(np.float64), grads[r].cpu().numpy().astype(np.float64)
        for f in range(F):
            t = full._feat_table[f]
            for b in range(B):
                s, e = off[f * B + b], off[f * B + b + 1]
                for l in range(s, e):
                    sc = w[l] / W / ((e - s) if lay.pool[f] == 1 else 1)
                    want[t][ids[l]] += sc * g[b, lay.col[f]:lay.col[f] + D]
                    touched[t][ids[l]] = True
    _, G = _helpers()
    hot_rows = 0
    for t, c in enumerate(cfgs):
        got = G._gathered(groups, plan, cfgs, full, t).cpu().numpy()
        np.testing.assert_array_equal(got[touched[t]], want[t][touched[t]].astype(f32), err_msg=c.name)
        assert not got[~touched[t]].any(), c.name
        hot_rows += int(touched[t].sum())
    assert hot_rows > 0


def test_all_ones_weights_are_the_unweighted_peer_step(kernels):
    W, B = 3, 257
    M, cfgs, plan, spec, full = _setup(W, "adagrad", 4)
    rng = np.random.default_rng(5)
    F = len(full.feature_names())
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    batches = [_bags(rng, F, B, feat_rows) for _ in range(W)]
    grads = [torch.from_numpy(rng.standard_normal((B, F * 16)).astype(f32)).cuda() for _ in range(W)]
    ones = [torch.ones(b[0].numel(), device="cuda") for b in batches]
    g_w, o_w = _run(W, B, spec, full, cfgs, plan, batches, ones, grads, "ones")
    g_u, o_u = _run(W, B, spec, full, cfgs, plan, batches, None, grads, "plain")
    for s in range(2):
        for r in range(W):
            assert torch.equal(o_w[s][r], o_u[s][r]), (s, r)
    for a, b in zip(g_w, g_u):
        assert torch.equal(a.local.weights.data, b.local.weights.data)
        assert torch.equal(a.local.opt_state, b.local.opt_state)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_ccp_mmoe_two_gpus_peer_memory():
    """The Ali-CCP MMoE config (nine weighted features) sharded over peer memory on two GPUs against its unsharded
    twin (tests/test_distributed_cpu.py's comparison: logits, loss, updated tables, dense weights)."""
    from test_distributed_cpu import _run as run_sharded

    ccp = os.path.join(HERE, "golden", "ref_examples", "mmoe_taobao_ccp.config")
    run_sharded(2, ccp, "mixed", rw_min_rows=250, use_cuda=True, static_capacity=2.5, exchange="peer")
