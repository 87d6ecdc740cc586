"""N>1 on real GPUs (needs >= 2 devices: `python -m pytest tests/test_distributed_gpu.py` on a multi-GPU node):
the same sharded-vs-unsharded comparison as tests/test_distributed_cpu.py, but with the CUDA kernels as compute and
NCCL all-to-alls.  Skipped on single-GPU boxes."""
import pytest
import torch

from test_distributed_cpu import _run

pytestmark = pytest.mark.gpu
need2 = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")


@need2
@pytest.mark.parametrize("sharding", ["row_wise", "table_wise"])
def test_dlrm_two_gpus(sharding):
    _run(2, "dlrm_criteo", sharding, use_cuda=True)


@need2
def test_deepfm_mixed_two_gpus():
    _run(2, "deepfm_criteo", "mixed", rw_min_rows=200, use_cuda=True)


@need2
def test_din_sequence_two_gpus():
    _run(2, "multi_tower_din_taobao", "mixed", rw_min_rows=250, use_cuda=True)


@need2
@pytest.mark.parametrize("sharding", ["row_wise", "mixed"])
def test_dlrm_two_gpus_peer_memory(sharding):
    """exchange="peer": requester-side gather over NVLink, owner-side pull, barrier kernels — same checks against the
    unsharded twin as the NCCL path (logits, loss, updated tables, dense weights)."""
    _run(2, "dlrm_criteo", sharding, rw_min_rows=200 if sharding == "mixed" else 0, use_cuda=True, static_capacity=2.5,
         exchange="peer")


@need2
@pytest.mark.parametrize("name,sharding,rw_min_rows", [("deepfm_criteo", "table_wise", 0), ("mmoe_taobao", "mixed", 250),
                                                       ("multi_tower_din_taobao", "mixed", 250),
                                                       ("multi_tower_din_taobao", "table_wise", 0)])
def test_baseline_configs_two_gpus_peer_memory(name, sharding, rw_min_rows):
    """BASELINE.json configs[2..4] over peer memory: DeepFM table-wise (two dim groups: D=4 wide + D=16), MMoE mixed
    table-wise + row-wise, DIN with its un-pooled sequence collection (ragged, device-side: no host read of split
    sizes anywhere)."""
    _run(2, name, sharding, rw_min_rows=rw_min_rows, use_cuda=True, static_capacity=2.5, exchange="peer")


@need2
def test_dlrm_two_gpus_peer_memory_sparse_adam():
    _run(2, "dlrm_criteo", "row_wise", use_cuda=True, static_capacity=2.5, exchange="peer", sparse_opt="adam")
