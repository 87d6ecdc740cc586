"""[EXT] known-answer vectors for the third-party half of the path, restated from the upstream projects' own unit tests
and docstrings (torchrec 1.x / fbgemm_gpu 1.x — the wheels the reference pins in requirements/runtime.txt:5,25; their
sources are not part of the reference and cannot be installed offline, so these are written down from the published
material, each with the upstream symbol it comes from).  Every vector was re-derived by hand from the documented
semantics when it was added (the derivation is in the comment) — a vector that only restated this repo's own reading
would prove nothing.

TEST INFRASTRUCTURE: used by tests/test_ext_vectors.py to pin oracle/tzk_oracle.py (and, on a GPU, the CUDA kernels).
"""

# ---------------------------------------------------------------------------------------------------------------------
# fbgemm_gpu  sparse_ops: block_bucketize_sparse_features — upstream test
# fbgemm_gpu/test/sparse/block_bucketize_test.py::BlockBucketizeTest::test_block_bucketize_sparse_features
# (sequence=True, bucketize_pos=False; T = 4 features, B = 2, my_size = 2 buckets, per-feature block sizes).
# Derivation: bucket = id // block_size[t], new id = id % block_size[t], output lengths laid out [bucket][t][b], ids of a
# (bucket, t, b) cell keep their order; unbucketize_permute[i] = new position of original position i.
#   t0 (bs 5):  b1 [3,4]           -> bucket 0: 3,4
#   t1 (bs 15): b0 [15]  b1 [11,28,29] -> 15 -> (1,0); 11 -> (0,11); 28 -> (1,13); 29 -> (1,14)
#   t2 (bs 10): b0 [1,10] b1 [11,12,13] -> 1 -> (0,1); 10 -> (1,0); 11,12,13 -> (1, 1..3)
#   t3 (bs 20): b0 [11,22,20] b1 [20]   -> 11 -> (0,11); 22 -> (1,2); 20 -> (1,0); 20 -> (1,0)
FBGEMM_BLOCK_BUCKETIZE = dict(
    lengths=[0, 2, 1, 3, 2, 3, 3, 1],
    indices=[3, 4, 15, 11, 28, 29, 1, 10, 11, 12, 13, 11, 22, 20, 20],
    block_sizes=[5, 15, 10, 20],
    my_size=2, T=4, B=2,
    new_lengths=[0, 2, 0, 1, 1, 0, 1, 0, 0, 0, 1, 2, 1, 3, 2, 1],
    new_indices=[3, 4, 11, 1, 11, 0, 13, 14, 0, 1, 2, 3, 2, 0, 0],
    unbucketize_permute=[0, 1, 5, 2, 6, 7, 3, 8, 9, 10, 11, 4, 12, 13, 14],
)

# ---------------------------------------------------------------------------------------------------------------------
# torchrec.sparse.jagged_tensor.KeyedJaggedTensor — class docstring ("Feature0": [V0,V1] None [V2]; "Feature1": [V3] [V4]
# [V5,V6,V7]): the key-major layout of SURVEY App. A.1.
TORCHREC_KJT_DOC = dict(
    keys=["Feature0", "Feature1"],
    values=[0, 1, 2, 3, 4, 5, 6, 7],
    lengths=[2, 0, 1, 1, 1, 3],
    offsets=[0, 2, 2, 3, 4, 5, 8],
    stride=3,
    length_per_key=[3, 5],
    offset_per_key=[0, 3, 8],
    # kjt.permute([1, 0]): whole per-key segments swap (fbgemm::permute_2D_sparse_data); derived from the layout above
    permuted_keys=["Feature1", "Feature0"],
    permuted_values=[3, 4, 5, 6, 7, 0, 1, 2],
    permuted_lengths=[1, 1, 3, 2, 0, 1],
)

# ---------------------------------------------------------------------------------------------------------------------
# torchrec.sparse.jagged_tensor.JaggedTensor.to_padded_dense — method docstring
# (values 1..8, offsets [0,2,2,3,4,5,8]; default desired_length = longest row, padding 0; then desired_length=2, padding 10)
TORCHREC_TO_PADDED_DENSE_DOC = dict(
    values=[1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0],
    offsets=[0, 2, 2, 3, 4, 5, 8],
    dense_default=[[1.0, 2.0, 0.0], [0.0, 0.0, 0.0], [3.0, 0.0, 0.0], [4.0, 0.0, 0.0], [5.0, 0.0, 0.0], [6.0, 7.0, 8.0]],
    dense_len2_pad10=[[1.0, 2.0], [10.0, 10.0], [3.0, 10.0], [4.0, 10.0], [5.0, 10.0], [6.0, 7.0]],
)

# ---------------------------------------------------------------------------------------------------------------------
# torchrec.sparse.jagged_tensor.KeyedTensor — class docstring: two [3, 2] tensors of ones / twos under keys
# "Embedding A", "Embedding B" (key_dim = 1); regroup is the column gather of App. A.13.
TORCHREC_KEYED_TENSOR_DOC = dict(
    keys=["Embedding A", "Embedding B"],
    length_per_key=[2, 2],
    values=[[1.0, 1.0, 2.0, 2.0]] * 3,
    offset_per_key=[0, 2, 4],
    embedding_b=[[2.0, 2.0]] * 3,
    # KeyedTensor.regroup([kt], [["Embedding B", "Embedding A"], ["Embedding A"]]) — derived
    regroup_groups=[["Embedding B", "Embedding A"], ["Embedding A"]],
    regrouped=[[[2.0, 2.0, 1.0, 1.0]] * 3, [[1.0, 1.0]] * 3],
)

# ---------------------------------------------------------------------------------------------------------------------
# torchrec.distributed.sharding.rw_sharding / embedding_sharding.bucketize_kjt_before_all2all: row-wise shard geometry
# block_size = ceil(hash_size / world_size), the last shard is short, ranks beyond the table are empty (App. A.7;
# torchrec.distributed.sharding_plan._get_parameter_size_offsets / row_wise()).  Hand-derived from that rule for the
# edge cases SURVEY §8c(5) names: hash_size % W != 0 (39060 rows over 8 ranks) and tables smaller than W (3 and 4 rows).
TORCHREC_RW_GEOMETRY = [
    # (hash_size, W, block, rows per rank)
    (39060, 8, 4883, [4883, 4883, 4883, 4883, 4883, 4883, 4883, 4879]),
    (3, 8, 1, [1, 1, 1, 0, 0, 0, 0, 0]),
    (4, 8, 1, [1, 1, 1, 1, 0, 0, 0, 0]),
    (10, 4, 3, [3, 3, 3, 1]),
    (40000000, 8, 5000000, [5000000] * 8),
]

# ---------------------------------------------------------------------------------------------------------------------
# torch.nn.functional.embedding_bag — PyTorch documentation example (sum mode is what EmbeddingBagCollection pools
# with; the unsharded torchrec EBC on CPU dispatches to exactly this op).  weight = 10 x 3 table with row r = [r, r, r]
# chosen here so that the expected sums can be read off: bags [1,2,4,5] and [4,3,2,9] -> 12 and 18.
EMBEDDING_BAG_DOC_SHAPE = dict(
    input=[1, 2, 4, 5, 4, 3, 2, 9], offsets=[0, 4], rows=10, dim=3,
    sum=[[12.0] * 3, [18.0] * 3], mean=[[3.0] * 3, [4.5] * 3],
)
