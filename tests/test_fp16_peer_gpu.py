"""FP16 tables (data_type = FP16) on the peer-memory sparse step, on ONE GPU: W virtual ranks are threads of this process
whose "symmetric" buffers are allocations of the same device (tests/test_peer_gpu.py's setup) — the CUDA kernels through
the C-ABI, `PeerState`, side streams.  Checked against the unsharded FP16 CUDA collection:
  * every rank's forward has the bits of tzk_pooled_gather_fwd_f16, tzk_pooled_gather_fwd_weighted (f16) and
    tzk_seq_gather_fwd_f16, with the one-launch and the split gather;
  * tables after two steps of every sparse optimizer, push and pull transport: within one fp16 ulp of the unsharded
    FP16 step on the concatenated batch (grad / W); with dyadic data (SGD, lr = -1, zero arena) bit-identical halfs;
  * a graphed FP16 peer step (one rank) replays the eager step bit for bit.
Two real GPUs: DLRM-Criteo with every table FP16, peer exchange, against its unsharded FP16 twin."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

pytestmark = pytest.mark.gpu
f32 = np.float32

OPTIMIZERS = ["sgd", "adagrad", "rowwise_adagrad", "adam", "partial_rowwise_adam", "lamb", "partial_rowwise_lamb",
              "lars_sgd"]


def _helpers():
    import test_peer_exchange_model as M
    import test_peer_gpu as G

    return M, G


def _fp16_bag_configs():
    M, _ = _helpers()
    from torcheasyrec_b200.embedding_modules import DataType, EmbeddingBagConfig

    return [EmbeddingBagConfig(num_embeddings=c.num_embeddings, embedding_dim=c.embedding_dim, name=c.name,
                               feature_names=list(c.feature_names), pooling=c.pooling, data_type=DataType.FP16)
            for c in M._pooled_configs()]


def _setup(W, opt, seed, lr=0.05):
    from torcheasyrec_b200.distributed import TABLE_WISE, make_plan
    from torcheasyrec_b200.embedding_modules import EmbeddingBagCollection, SparseOptimizerSpec

    torch.manual_seed(seed)
    cfgs = _fp16_bag_configs()     # SUM / MEAN, a shared table, a 2-row table, a table-wise one; small ones mirrored
    plan = make_plan(cfgs, W, "row_wise", {"t_tw": [TABLE_WISE], "t_tiny": [TABLE_WISE]})
    spec = SparseOptimizerSpec.from_name(opt, lr=lr)
    full = EmbeddingBagCollection(cfgs, device="cuda")
    full.set_optimizer(spec)
    assert full.weights.dtype == torch.float16
    return cfgs, plan, spec, full


def _bags(rng, F, B, feat_rows, lens_from=(0, 1, 2, 3, 4)):
    lens = rng.choice(list(lens_from), F * B)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ids = np.concatenate([rng.integers(0, feat_rows[b // B], lens[b]) for b in range(F * B)] + [np.zeros(0, np.int64)])
    return torch.from_numpy(ids.astype(np.int64)).cuda(), torch.from_numpy(off).cuda()


def _run(W, B, spec, full, cfgs, plan, batches, weights, grads, tag, steps=2, pooled=True, budget=None):
    M, G = _helpers()
    from torcheasyrec_b200 import peer_exchange

    F = len(full.feature_names())
    groups = G._seed_groups(cfgs, plan, W, pooled, full, spec, 2.5)
    assert all(g.local.weights.dtype == torch.float16 for g in groups)
    registry, outs = {}, [[None] * W for _ in range(steps)]

    def body(r, tbar):
        torch.cuda.set_device(0)

        class St(M._sim_mixin(registry, tbar, tag, "cuda"), peer_exchange.PeerState):
            pass

        st = St(groups[r], plan, None, B, budget or [B * 4] * F)
        assert st.tables.t.dtype == torch.float16 and (st.mirror is None or st.mirror.dtype == torch.float16)
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


def _within_one_ulp(got, want, msg):
    from fp16_sharded_ref import assert_within_one_ulp

    assert got.dtype == torch.float16 and want.dtype == torch.float16
    assert_within_one_ulp(got.cpu().numpy(), want.cpu().numpy(), msg)


@pytest.mark.parametrize("split", ["0", "1"])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("B", [64, 4099])
def test_fp16_peer_forward_is_the_unsharded_f16_gather(kernels, monkeypatch, B, weighted, split):
    monkeypatch.setenv("TZK_PEER_SPLIT_GATHER", split)
    W = 3
    cfgs, plan, spec, full = _setup(W, "adagrad", 1)
    rng = np.random.default_rng(B + int(split) + 2 * weighted)
    F = len(full.feature_names())
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    batches = [_bags(rng, F, B, feat_rows) for _ in range(W)]
    weights = ([torch.from_numpy(rng.standard_normal(b[0].numel()).astype(f32)).cuda() for b in batches]
               if weighted else None)
    _, outs = _run(W, B, spec, full, cfgs, plan, batches, weights, None, f"fwd{split}{weighted}", steps=1)
    for r in range(W):
        kw = {} if weights is None else {"per_sample_weights": weights[r]}
        want = kernels.pooled_gather_fwd(full.weights.data, full.layout, batches[r][0], batches[r][1], B, **kw)
        assert torch.equal(outs[0][r], want), r


@pytest.mark.parametrize("bwd", ["push", "pull"])
@pytest.mark.parametrize("opt", OPTIMIZERS)
def test_fp16_peer_tables_match_unsharded(kernels, monkeypatch, opt, bwd):
    monkeypatch.setenv("TZK_PEER_BWD", bwd)
    M, _ = _helpers()
    W, B, D = 4, 1000, 16
    cfgs, plan, spec, full = _setup(W, opt, 2)
    rng = np.random.default_rng(17)
    F = len(full.feature_names())
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    batches = [_bags(rng, F, B, feat_rows) for _ in range(W)]
    grads = [torch.from_numpy(rng.standard_normal((B, F * D)).astype(f32)).cuda() for _ in range(W)]
    groups, outs = _run(W, B, spec, full, cfgs, plan, batches, None, grads, f"tab{opt}{bwd}")
    cat = M._cat_key_major([b[0].cpu() for b in batches], [b[1].cpu() for b in batches], F, B, W)
    cat_ids, cat_off = cat[0].cuda(), cat[1].cuda()
    cat_grad = torch.cat(grads) / W
    for step in range(2):
        if step == 0:
            for r in range(W):
                want = kernels.pooled_gather_fwd(full.weights.data, full.layout, batches[r][0], batches[r][1], B)
                assert torch.equal(outs[0][r], want)
        kernels.fused_bwd(spec.kind, True, cat_grad, full.weights.data, full.opt_state, full.layout, cat_ids, cat_off,
                          B * W, spec.lr, spec.eps, 1.0, **full.opt_extras())
    _, G = _helpers()
    for t, c in enumerate(cfgs):
        _within_one_ulp(G._gathered(groups, plan, cfgs, full, t), full.table_weight(t), f"{opt}/{bwd} {c.name}")


@pytest.mark.parametrize("bwd", ["push", "pull"])
@pytest.mark.parametrize("W", [2, 4])
def test_fp16_peer_dyadic_step_is_bit_identical(kernels, monkeypatch, W, bwd):
    """SGD, lr = -1, zero arena, dyadic gradients / bag lengths / W: every row's fp32 gradient sum is exact on both
    sides, so the rounded half rows must be the same bits as the unsharded FP16 step's."""
    monkeypatch.setenv("TZK_PEER_BWD", bwd)
    M, G = _helpers()
    B, D = 4099, 16
    cfgs, plan, spec, full = _setup(W, "sgd", 3, lr=-1.0)
    full.weights.data.zero_()
    rng = np.random.default_rng(29 + W)
    F = len(full.feature_names())
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    batches = [_bags(rng, F, B, feat_rows, lens_from=(0, 1, 2, 4)) for _ in range(W)]
    grads = [torch.from_numpy((rng.integers(-8, 9, (B, F * D)) / 8.0).astype(f32)).cuda() for _ in range(W)]
    groups, _ = _run(W, B, spec, full, cfgs, plan, batches, None, grads, f"dy{W}{bwd}", steps=1)
    cat = M._cat_key_major([b[0].cpu() for b in batches], [b[1].cpu() for b in batches], F, B, W)
    kernels.fused_bwd(spec.kind, True, torch.cat(grads) / W, full.weights.data, full.opt_state, full.layout,
                      cat[0].cuda(), cat[1].cuda(), B * W, spec.lr, spec.eps, 1.0, **full.opt_extras())
    moved = 0
    for t, c in enumerate(cfgs):
        got, want = G._gathered(groups, plan, cfgs, full, t), full.table_weight(t)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), c.name
        moved += int((want != 0).any(dim=1).sum())
    assert moved > 0


@pytest.mark.parametrize("W", [2, 3])
def test_fp16_peer_sequence_step_on_one_gpu(kernels, W):
    M, G = _helpers()
    from torcheasyrec_b200.distributed import TABLE_WISE, make_plan
    from torcheasyrec_b200.embedding_modules import DataType, EmbeddingCollection, EmbeddingConfig, SparseOptimizerSpec

    rng = np.random.default_rng(11 + W)
    mk = lambda n, rows, feats: EmbeddingConfig(num_embeddings=rows, embedding_dim=16, name=n, feature_names=feats,
                                                data_type=DataType.FP16)
    cfgs = [mk("q", 50, ["q_id"]), mk("s1", 21100, ["seq_a"]), mk("s2", 40, ["seq_b"])]
    B, D, max_len = 300, 16, 20
    plan = make_plan(cfgs, W, "row_wise", {"s2": [TABLE_WISE]})
    spec = SparseOptimizerSpec.from_name("adagrad", lr=0.1)
    full = EmbeddingCollection(cfgs, device="cuda")
    full.set_optimizer(spec)
    F = len(full.feature_names())
    feat_rows = [cfgs[t].num_embeddings for t in full._feat_table]
    batches = []
    for _ in range(W):
        lens = np.concatenate([np.ones(B, np.int64), rng.integers(0, max_len + 1, B), rng.integers(0, max_len + 1, B)])
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        idv = np.concatenate([rng.integers(0, feat_rows[b // B], lens[b]) for b in range(F * B)]).astype(np.int64)
        batches.append((torch.from_numpy(idv).cuda(), torch.from_numpy(off).cuda()))
    grads = [torch.from_numpy(rng.standard_normal((b[0].numel(), D)).astype(f32)).cuda() for b in batches]
    groups, outs = _run(W, B, spec, full, cfgs, plan, batches, None, grads, f"seq{W}", steps=1, pooled=False,
                        budget=[B, B * max_len, B * max_len])
    for r in range(W):
        assert torch.equal(outs[0][r], kernels.seq_gather_fwd(full.weights.data, full.layout, *batches[r], B))
    ids, offs = [b[0].cpu() for b in batches], [b[1].cpu() for b in batches]
    cat_ids, cat_off = M._cat_key_major(ids, offs, F, B, W)
    rows = [grads[r][offs[r][f * B]:offs[r][(f + 1) * B]] for f in range(F) for r in range(W)]
    kernels.fused_bwd(spec.kind, False, torch.cat(rows) / W, full.weights.data, full.opt_state, full.layout,
                      cat_ids.cuda(), cat_off.cuda(), B * W, spec.lr, spec.eps, 1.0)
    for t, c in enumerate(cfgs):
        _within_one_ulp(G._gathered(groups, plan, cfgs, full, t), full.table_weight(t), c.name)


def _graph_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    try:
        from fp16_sharded_ref import fp16_edits

        from torcheasyrec_b200.engine import GraphedTrainStep, Pipeline

        mk = lambda: Pipeline("dlrm_criteo", device=f"cuda:{rank}", max_rows=5000, seed=3, sharding="row_wise",
                              exchange="peer", static_capacity=2.5, edits=fp16_edits("dlrm_criteo"))
        a = mk()
        batches = [a.synthetic_batch(1024, seed=40 + i + 10 * rank) for i in range(4)]
        step = GraphedTrainStep(a, batches[0], warmup=3)       # the warm-up steps already trained `a` a little
        b = mk()                                               # the eager twin, cloned AFTER the capture
        for ca, cb in zip(a.model.sparse_collections(), b.model.sparse_collections()):
            assert ca.weights.dtype == torch.float16
            cb.weights.data.copy_(ca.weights.data)
            cb.opt_state.copy_(ca.opt_state)
        da = dict((n, p) for n, p in a.model.named_parameters() if not n.endswith("weights"))
        with torch.no_grad():
            for n, p in b.model.named_parameters():
                if n in da:
                    p.copy_(da[n])
        b.dense_optimizer.load_state_dict(copy.deepcopy(a.dense_optimizer.state_dict()))
        la, lb = [], []
        for bt in batches[1:]:
            step.load(bt.pin_memory())
            la.append(float(step.replay()))
            lb.append(float(b.eager_step(bt.to(f"cuda:{rank}"))))
        np.testing.assert_allclose(la, lb, rtol=1e-6)
        for ca, cb in zip(a.model.sparse_collections(), b.model.sparse_collections()):
            assert torch.equal(ca.weights.data.view(torch.int16), cb.weights.data.view(torch.int16))
            assert torch.equal(ca.opt_state, cb.opt_state)
        for sm in a.sharded:
            sm.check_overflow()
        q.put((rank, "ok"))
    except Exception:
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def _spawn(world, target):
    import torch.multiprocessing as mp
    from test_distributed_cpu import _free_port

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=900) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    bad = [(r, m) for r, m in res if m != "ok"]
    assert not bad, "\n".join(f"rank {r}: {m}" for r, m in bad)


def test_fp16_peer_graphed_step_equals_eager_step():
    """DLRM-Criteo with FP16 tables on the peer exchange (one rank): the captured step replays the eager step — losses,
    half tables and Adagrad state bit for bit."""
    _spawn(1, _graph_worker)


def _two_gpu_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    try:
        from fp16_sharded_ref import verify_fp16_sharded

        verify_fp16_sharded("dlrm_criteo", f"cuda:{rank}", "row_wise", exchange="peer", static_capacity=2.5)
        q.put((rank, "ok"))
    except Exception:
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_dlrm_fp16_two_gpus_peer_memory():
    """DLRM-Criteo (small hash sizes), every table data_type FP16, peer exchange at W = 2, against the unsharded FP16
    run on the concatenated batch: logits, loss, half tables within one ulp, dense parameters."""
    _spawn(2, _two_gpu_worker)
