"""DLRM-Criteo's interaction, wide layer, tower tail and BCE as one autograd node (dense_gemm.InteractWideTailFn, the
tail kernel in masked mode) against the two nodes it replaces (InteractWideFn, then _TowerTailFn): bit for bit for
loss.backward(), and for a loss gradient of 2.5 the gradients from dZ are those of 2.5 dZ and the wide layer's bias
gradient is its column sum times 2.5.  Then whole training steps of the model through either path."""
import pytest
import torch

pytestmark = pytest.mark.gpu
IN_MAP = ((0, 0, 351), (351, 352, 432))


def _inputs(B, seed):
    g = torch.Generator().manual_seed(seed)
    t = [torch.randn(B, 16, generator=g), torch.randn(B, 416, generator=g) * 0.5, torch.randn(64, 783, generator=g) / 28,
         torch.randn(64, generator=g) / 4, torch.randn(32, 64, generator=g) / 8, torch.randn(32, generator=g) / 10,
         torch.randn(1, 32, generator=g) / 6, torch.randn(1, generator=g) / 10]
    labels = (torch.rand(B, generator=g) < 0.25).float()
    return [x.cuda().requires_grad_(True) for x in t], labels.cuda()


def _run(fused, leaves, labels, scale):
    from torcheasyrec_b200 import dense_gemm as G

    dense, sparse, w, b, w1, b1, w2, b2 = [x.detach().clone().requires_grad_(True) for x in leaves]
    assert G.interact_wide_usable(dense, sparse, w, 26, 16)
    if fused:
        assert G.interact_wide_tail_usable(sparse, w1, w2, labels)
        loss, logits = G.InteractWideTailFn.apply(dense, sparse, w, b, IN_MAP, w1, b1, w2, b2, labels)
    else:
        y1 = G.InteractWideFn.apply(G._gemm3x_lib(), dense, sparse, w, b, IN_MAP)
        assert G.tower_tail_usable(y1, w1, w2, labels)
        loss, logits = G.tower_tail_bce(y1, w1, b1, w2, b2, labels)
    (loss if scale is None else scale * loss).backward()
    return loss.detach(), logits, [x.grad for x in (dense, sparse, w, b, w1, b1, w2, b2)]


@pytest.mark.parametrize("B", [65536, 1000])
def test_one_node_gives_the_two_nodes_bits(B):
    leaves, labels = _inputs(B, B)
    loss, logits, grads = _run(True, leaves, labels, None)
    loss0, logits0, grads0 = _run(False, leaves, labels, None)
    assert torch.equal(loss, loss0) and torch.equal(logits, logits0)
    for name, g, g0 in zip(("dense", "sparse", "w", "b", "w1", "b1", "w2", "b2"), grads, grads0):
        assert g is not None and torch.equal(g, g0), name


def test_loss_gradient_scales_dz_and_the_bias_gradient():
    leaves, labels = _inputs(65536, 11)
    _, _, grads1 = _run(True, leaves, labels, None)
    _, _, grads = _run(True, leaves, labels, 2.5)
    _, _, grads0 = _run(False, leaves, labels, 2.5)
    # d_dense, d_sparse, dW: the chain's mask(2.5 dy1) is 2.5 mask(dy1) exactly, so its kernels saw the same dZ
    for i in (0, 1, 2, 4, 5, 6, 7):
        assert torch.equal(grads[i], grads0[i]), i
    # db: colsum(dZ) * 2.5, one rounding (the chain sums 2.5 dZ instead)
    assert torch.equal(grads[3], grads1[3] * 2.5)
    torch.testing.assert_close(grads[3], grads0[3], rtol=1e-5, atol=1e-7)


def test_training_steps_match_the_two_node_chain(monkeypatch):
    from torcheasyrec_b200.engine import Pipeline
    from torcheasyrec_b200.rank_models import DLRM

    taken = []
    real = DLRM._interact_wide_tail

    def spy(self, *a):
        out = real(self, *a)
        taken.append(out is not None)
        return out

    monkeypatch.setattr(DLRM, "_interact_wide_tail", spy)
    new = Pipeline("dlrm_criteo", device="cuda", max_rows=200000, seed=7, capturable=False)
    old = Pipeline("dlrm_criteo", device="cuda", max_rows=200000, seed=7, capturable=False)
    old.model.load_state_dict(new.model.state_dict())
    old.model._interact_wide_tail = lambda *a: None                  # the parent's path: two nodes
    for step in range(2):
        batch = new.synthetic_batch(8192, seed=100 + step).to("cuda")
        l_new, l_old = new.eager_step(batch), old.eager_step(batch)
        assert torch.equal(l_new, l_old), step
    assert taken and all(taken)
    s_new, s_old = new.model.state_dict(), old.model.state_dict()
    assert s_new.keys() == s_old.keys()
    for k in s_new:
        assert torch.equal(s_new[k], s_old[k]), k
    for c_new, c_old in zip(new.model.sparse_collections(), old.model.sparse_collections()):
        assert torch.equal(c_new.dense_weights(), c_old.dense_weights())
