"""Generators for the pipeline configs BASELINE.json names (text format, same message tree as the reference's
examples/{dlrm_criteo,deepfm_criteo,mmoe_taobao,multi_tower_din_taobao,masknet_criteo,ple_taobao,
pepnet_taobao,rocket_launching_criteo,tdm_taobao}.config).

The package does not depend on the reference's files, so the configs are re-derived here from their defining facts
(SURVEY.md §8 / Appendix D): the Criteo hash sizes, the Taobao table list and price boundaries, and the model
blocks.  tests/test_config.py checks, against copies stored under tests/golden/ref_examples/, that each generated
config parses to the same tree as the reference's example file — i.e. the reference's own
examples/*.config load unchanged through `config.load_pipeline_config` and mean the same thing.
"""

from typing import List, Optional, Sequence

CRITEO_HASH_SIZES = [40000000, 39060, 17295, 7424, 20265, 3, 7122, 1543, 63, 40000000, 3067956, 405282, 10, 2209,
                     11938, 155, 4, 976, 14, 40000000, 40000000, 40000000, 590152, 12973, 108, 36]

TAOBAO_USER = [("user_id", 1141730), ("cms_segid", 98), ("cms_group_id", 14), ("final_gender_code", 3),
               ("age_level", 8), ("pvalue_level", 5), ("shopping_level", 5), ("occupation", 3),
               ("new_user_class_level", 6)]
TAOBAO_ITEM = [("adgroup_id", 846812), ("cate_id", 12961), ("campaign_id", 423438), ("customer", 255877),
               ("brand", 461498)]
TAOBAO_PRICE_BOUNDARIES = [
    1.1, 2.2, 3.6, 5.2, 7.39, 9.5, 10.5, 12.9, 15, 17.37, 19, 20, 23.8, 25.8, 28, 29.8, 31.5, 34, 36, 38, 39, 40,
    45, 48, 49, 51.6, 55.2, 58, 59, 63.8, 68, 69, 72, 78, 79, 85, 88, 90, 97.5, 98, 99, 100, 108, 115, 118, 124,
    128, 129, 138, 139, 148, 155, 158, 164, 168, 171.8, 179, 188, 195, 198, 199, 216, 228, 238, 248, 258, 268, 278,
    288, 298, 299, 316, 330, 352, 368, 388, 398, 399, 439, 478, 499, 536, 580, 599, 660, 699, 780, 859, 970, 1080,
    1280, 1480, 1776, 2188, 2798, 3680, 5160, 8720]


def _header(train: str, evalp: str, model_dir: str, fg_mode: str, labels: Sequence[str], eval_steps: Optional[int],
            batch_size: int = 8192, quota: bool = True) -> str:
    ev = f"    num_steps: {eval_steps}\n" if eval_steps else ""
    lab = "".join(f'    label_fields: "{x}"\n' for x in labels)
    return (f'train_input_path: "odps://{{PROJECT}}/tables/{train}"\n'
            f'eval_input_path: "odps://{{PROJECT}}/tables/{evalp}"\n'
            f'model_dir: "experiments/{model_dir}"\n'
            "train_config {\n"
            "    sparse_optimizer {\n        adagrad_optimizer {\n            lr: 0.001\n        }\n"
            "        constant_learning_rate {\n        }\n    }\n"
            "    dense_optimizer {\n        adam_optimizer {\n            lr: 0.001\n        }\n"
            "        constant_learning_rate {\n        }\n    }\n"
            "    num_epochs: 1\n}\n"
            f"eval_config {{\n{ev}}}\n"
            f"data_config {{\n    batch_size: {batch_size}\n    dataset_type: OdpsDataset\n    fg_mode: {fg_mode}\n"
            f'{lab}' + ('    odps_data_quota_name: ""\n' if quota else "") + "    num_workers: 8\n}\n")


def _id_feature(name: str, side: Optional[str], rows: int, dim: int = 16, field: str = "num_buckets") -> str:
    expr = f'        expression: "{side}:{name}"\n' if side else ""
    return ("feature_configs {\n    id_feature {\n"
            f'        feature_name: "{name}"\n{expr}'
            f"        {field}: {rows}\n        embedding_dim: {dim}\n    }}\n}}\n")


def _group(name: str, feats: Sequence[str], gtype: str) -> str:
    names = "".join(f'        feature_names: "{f}"\n' for f in feats)
    return f'    feature_groups {{\n        group_name: "{name}"\n{names}        group_type: {gtype}\n    }}\n'


def _mlp(field: str, units: Sequence[int], indent: str) -> str:
    return f"{indent}{field} {{\n{indent}    hidden_units: [{', '.join(str(u) for u in units)}]\n{indent}}}\n"


def _criteo_features(fg: bool) -> str:
    """fg=True: FG_DAG flavour (expressions + log normaliser, dlrm); False: FG_NONE flavour (names only, deepfm)."""
    out = []
    for i in range(13):
        extra = (f'        expression: "user:int_{i}"\n        normalizer: "method=expression,expr=log(x+3)"\n'
                 if fg else "")
        out.append("feature_configs {\n    raw_feature {\n" f'        feature_name: "int_{i}"\n{extra}    }}\n}}\n')
    for i, h in enumerate(CRITEO_HASH_SIZES):
        out.append(_id_feature(f"cat_{i}", "user" if fg else None, h))
    return "".join(out)


def dlrm_criteo() -> str:
    """examples/dlrm_criteo.config: 13 raw + 26 id(D=16); groups dense/sparse; dlrm{dense 64-16, final 64-32}."""
    ints = [f"int_{i}" for i in range(13)]
    cats = [f"cat_{i}" for i in range(26)]
    return (_header("criteo_terabyte_train_hashed_v1", "criteo_terabyte_val_test_hashed_v1", "dlrm_criteo", "FG_DAG",
                    ["label"], 100)
            + _criteo_features(True)
            + "model_config {\n" + _group("dense", ints, "DEEP") + _group("sparse", cats, "DEEP")
            + "    dlrm {\n" + _mlp("dense_mlp", [64, 16], "        ") + _mlp("final", [64, 32], "        ")
            + "        arch_with_sparse: true\n    }\n    num_class: 1\n"
            "    metrics {\n        auc {}\n    }\n    losses {\n        binary_cross_entropy {}\n    }\n}\n")


def deepfm_criteo() -> str:
    """examples/deepfm_criteo.config: groups wide(WIDE)/fm/deep; deepfm{deep 512-256-128, final 64}."""
    ints = [f"int_{i}" for i in range(13)]
    cats = [f"cat_{i}" for i in range(26)]
    return (_header("criteo_terabyte_train_hashed_v1", "criteo_terabyte_val_test_hashed_v1", "deepfm_criteo",
                    "FG_NONE", ["label"], 100, quota=False)
            + _criteo_features(False)
            + "model_config {\n" + _group("wide", cats, "WIDE") + _group("fm", cats, "DEEP")
            + _group("deep", ints + cats, "DEEP")
            + "    deepfm {\n" + _mlp("deep", [512, 256, 128], "        ") + _mlp("final", [64], "        ")
            + "    }\n    metrics {\n        auc {}\n    }\n    losses {\n        binary_cross_entropy {}\n    }\n}\n")


def _wukong_layer() -> str:
    return ("        wukong_layers {\n            lcb_feature_num: 16\n            fmb_feature_num: 16\n"
            "            compressed_feature_num: 24\n" + _mlp("feature_num_mlp", [512], "            ") + "        }\n")


def wukong_criteo() -> str:
    """examples/wukong_criteo.config with ONE edit: dense_mlp [512, 256, 128] -> [512, 256, 16].

    The reference's file does not build in the reference itself: its bottom MLP ends at 128 while the sparse features
    have embedding_dim 16, and tzrec/models/wukong.py:81-84 requires the two to match ("dense mlp last hidden_unit must
    be the same sparse feature dim").  This repo raises the same exception on that file; this generator is the nearest
    config that builds.  Otherwise the DLRM-Criteo inputs and two WuKong layers (lcb 16, fmb 16, k 24, MLP 512), final
    512-64."""
    ints = [f"int_{i}" for i in range(13)]
    cats = [f"cat_{i}" for i in range(26)]
    return (_header("criteo_terabyte_train_hashed_v1", "criteo_terabyte_val_test_hashed_v1", "wukong_criteo", "FG_DAG",
                    ["label"], 100)
            + _criteo_features(True)
            + "model_config {\n" + _group("dense", ints, "DEEP") + _group("sparse", cats, "DEEP")
            + "    wukong {\n" + _mlp("dense_mlp", [512, 256, 16], "        ") + _wukong_layer() + _wukong_layer()
            + _mlp("final", [512, 64], "        ")
            + "    }\n    num_class: 1\n"
            "    metrics {\n        auc {}\n    }\n    losses {\n        binary_cross_entropy {}\n    }\n}\n")


def masknet_criteo() -> str:
    """examples/masknet_criteo.config: 13 raw features (embedding_dim 16, but no dense_emb, so 1 wide each) + 26 hashed
    id(D=16) in one DEEP group all_features of width 26 * 16 + 13 = 429; mask_net{3 parallel blocks, reduction_ratio 3,
    hidden_dim 512, top_mlp 256-128-64}.  Unlike the other Criteo examples: empty paths, lr 1e-4 for both optimizers,
    save_checkpoints_epochs 1, no eval num_steps and no odps_data_quota_name."""
    ints = [f"int_{i}" for i in range(13)]
    cats = [f"cat_{i}" for i in range(26)]
    hdr = _header("", "", "", "FG_DAG", ["label"], None, quota=False)
    hdr = (hdr.replace('"odps://{PROJECT}/tables/"', '""').replace('"experiments/"', '""')
           .replace("lr: 0.001\n", "lr: 0.0001\n")
           .replace("    num_epochs: 1\n", "    num_epochs: 1\n    save_checkpoints_epochs: 1\n"))
    feats = []
    for i in range(13):
        feats.append("feature_configs {\n    raw_feature {\n" f'        feature_name: "int_{i}"\n'
                     f'        embedding_dim: 16\n        expression: "user:int_{i}"\n'
                     '        normalizer: "method=expression,expr=log(x+3)"\n    }\n}\n')
    for i, h in enumerate(CRITEO_HASH_SIZES):
        feats.append(_id_feature(f"cat_{i}", "item", h, field="hash_bucket_size"))
    return (hdr + "".join(feats)
            + "model_config {\n" + _group("all_features", cats + ints, "DEEP")
            + "    mask_net {\n        mask_net_module {\n            n_mask_blocks: 3\n"
            "            mask_block {\n                reduction_ratio: 3\n                hidden_dim: 512\n"
            "            }\n            use_parallel: true\n" + _mlp("top_mlp", [256, 128, 64], "            ")
            + "        }\n    }\n"
            "    metrics {\n        auc {}\n    }\n    losses {\n        binary_cross_entropy {}\n    }\n}\n")


def _taobao_features() -> str:
    out = [_id_feature(n, "user", r) for n, r in TAOBAO_USER] + [_id_feature(n, "item", r) for n, r in TAOBAO_ITEM]
    bounds = ", ".join(repr(float(b)) for b in TAOBAO_PRICE_BOUNDARIES)
    out.append('feature_configs {\n    raw_feature {\n        feature_name: "price"\n        expression: "item:price"\n'
               f"        boundaries: [{bounds}]\n        embedding_dim: 16\n    }}\n}}\n")
    out.append(_id_feature("pid", "context", 20, field="hash_bucket_size"))
    return "".join(out)


TAOBAO_FEATURE_NAMES = [n for n, _ in TAOBAO_USER] + [n for n, _ in TAOBAO_ITEM] + ["price", "pid"]
# mmoe_taobao lists `pid` between the user and the item features in its single group
TAOBAO_MMOE_ORDER = [n for n, _ in TAOBAO_USER] + ["pid"] + [n for n, _ in TAOBAO_ITEM] + ["price"]


def _task_tower(name: str, label: str, thresholds: Optional[int]) -> str:
    auc = f"auc {{ thresholds: {thresholds} }}" if thresholds else "auc {}"
    return ("        task_towers {\n"
            f'            tower_name: "{name}"\n            label_name: "{label}"\n'
            + _mlp("mlp", [256, 128, 64], "            ")
            + f"            metrics {{\n                {auc}\n            }}\n"
            "            losses {\n                binary_cross_entropy {}\n            }\n        }\n")


def mmoe_taobao() -> str:
    """examples/mmoe_taobao.config: 16 features in group `all`; 3 experts 512-256-128; towers ctr/cvr."""
    return (_header("taobao_multitask_sample_v1_train", "taobao_multitask_sample_v1/ds=20170513", "mmoe_taobao",
                    "FG_DAG", ["clk", "buy"], None, quota=False)
            + _taobao_features()
            + "model_config {\n" + _group("all", TAOBAO_MMOE_ORDER, "DEEP")
            + "    mmoe {\n" + _mlp("expert_mlp", [512, 256, 128], "        ") + "        num_expert: 3\n"
            + _task_tower("ctr", "clk", None) + _task_tower("cvr", "buy", 1000) + "    }\n}\n")


def _extraction_network(name: str, n: int, units: Sequence[int]) -> str:
    return ("        extraction_networks {\n" f'            network_name: "{name}"\n'
            f"            expert_num_per_task: {n}\n            share_num: {n}\n"
            + _mlp("task_expert_net", units, "            ") + _mlp("share_expert_net", units, "            ")
            + "        }\n")


def ple_taobao() -> str:
    """examples/ple_taobao.config: mmoe_taobao's features, group `all` and towers ctr/cvr; ple{3 extraction networks:
    2 + 2 experts 1024-512-256, 3 + 3 experts 256-128-64, 4 + 4 experts 128-64-32 (per task + shared)}."""
    return (_header("taobao_multitask_sample_v1_train", "taobao_multitask_sample_v1/ds=20170513", "ple_taobao",
                    "FG_DAG", ["clk", "buy"], None, quota=False)
            + _taobao_features()
            + "model_config {\n" + _group("all", TAOBAO_MMOE_ORDER, "DEEP")
            + "    ple {\n" + _extraction_network("layer1", 2, [1024, 512, 256])
            + _extraction_network("layer2", 3, [256, 128, 64]) + _extraction_network("layer3", 4, [128, 64, 32])
            + _task_tower("ctr", "clk", None) + _task_tower("cvr", "buy", 1000) + "    }\n}\n")


def pepnet_taobao() -> str:
    """examples/pepnet_taobao.config: mmoe_taobao's features and towers ctr/cvr, `occupation` also a label; groups all
    (mmoe_taobao's 16), domain (occupation), uia (13 user and item features); pepnet{3 domains by occupation, PPNet
    512-256 with dropout 0.1}; cvr weighs its loss by the clk task space (in 1, out 0)."""
    uia = ["user_id", "cms_segid", "cms_group_id", "final_gender_code", "age_level", "pvalue_level", "shopping_level",
           "new_user_class_level", "adgroup_id", "cate_id", "campaign_id", "brand", "price"]
    cvr = _task_tower("cvr", "buy", 1000)
    cvr = cvr[:cvr.rindex("        }\n")] + ('            task_space_indicator_label: "clk"\n'
                                           "            in_task_space_weight: 1\n"
                                           "            out_task_space_weight: 0\n        }\n")
    return (_header("taobao_multitask_sample_v1_train", "taobao_multitask_sample_v1/ds=20170513", "pepnet_taobao",
                    "FG_DAG", ["clk", "buy", "occupation"], None, quota=False)
            + _taobao_features()
            + "model_config {\n" + _group("all", TAOBAO_MMOE_ORDER, "DEEP") + _group("domain", ["occupation"], "DEEP")
            + _group("uia", uia, "DEEP")
            + "    pepnet {\n        domain_input_name: 'occupation'\n        task_domain_num: 3\n"
            "        ppnet_hidden_units: [512, 256]\n        ppnet_dropout_ratio: [0.1, 0.1]\n"
            + _task_tower("ctr", "clk", None) + cvr + "    }\n}\n")


def multi_tower_din_taobao() -> str:
    """examples/multi_tower_din_taobao.config: group deep (16) + SEQUENCE group seq (3 queries + click_50_seq)."""
    seq_feats = "".join(
        "        features {\n            id_feature {\n"
        f'                feature_name: "{n}"\n                expression: "item:{n}"\n'
        f"                num_buckets: {r}\n                embedding_dim: 16\n            }}\n        }}\n"
        for n, r in [("adgroup_id", 846812), ("cate_id", 12961), ("brand", 461498)])
    seq = ('feature_configs {\n    sequence_feature {\n        sequence_name: "click_50_seq"\n'
           '        sequence_length: 100\n        sequence_delim: "|"\n' + seq_feats + "    }\n}\n")
    seq_group = ["adgroup_id", "cate_id", "brand", "click_50_seq__adgroup_id", "click_50_seq__cate_id",
                 "click_50_seq__brand"]
    return (_header("taobao_multitask_sample_v1_train", "taobao_multitask_sample_v1/ds=20170513",
                    "multi_tower_din_taobao", "FG_DAG", ["clk"], None, quota=False)
            + _taobao_features() + seq
            + "model_config {\n" + _group("deep", TAOBAO_FEATURE_NAMES, "DEEP") + _group("seq", seq_group, "SEQUENCE")
            + "    multi_tower_din {\n        towers {\n            input: 'deep'\n"
            + _mlp("mlp", [512, 256, 128], "            ") + "        }\n        din_towers {\n            input: 'seq'\n"
            + _mlp("attn_mlp", [256, 64], "            ") + "        }\n" + _mlp("final", [64], "        ")
            + "    }\n    metrics {\n        auc {}\n    }\n    losses {\n        binary_cross_entropy {}\n    }\n}\n")


def _dbmtl_towers(thresholds: int, loss: str, num_class: str = "") -> str:
    def tower(name, label, auc, extra=""):
        return ("        task_towers {\n"
                f'            tower_name: "{name}"\n            label_name: "{label}"\n{num_class}'
                + _mlp("mlp", [256, 128, 64], "            ")
                + f"            metrics {{\n                {auc}\n            }}\n"
                f"            losses {{\n                {loss}\n            }}\n{extra}        }}\n")
    rel = '            relation_tower_names: "ctr"\n' + _mlp("relation_mlp", [64], "            ")
    return tower("ctr", "clk", "auc {}") + tower("cvr", "buy", f"auc {{ thresholds: {thresholds} }}", rel)


def dbmtl_taobao() -> str:
    """examples/dbmtl_taobao.config: mmoe_taobao's features and group `all`; dbmtl{bottom MLP 512; towers ctr and cvr
    with MLP 256-128-64, cvr related to ctr through a relation MLP 64}."""
    return (_header("taobao_multitask_sample_v1_train", "taobao_multitask_sample_v1/ds=20170513", "dbmtl_taobao",
                    "FG_DAG", ["clk", "buy"], None, quota=False)
            + _taobao_features()
            + "model_config {\n" + _group("all", TAOBAO_MMOE_ORDER, "DEEP")
            + "    dbmtl {\n" + _mlp("bottom_mlp", [512], "        ")
            + _dbmtl_towers(1000, "binary_cross_entropy {}") + "    }\n}\n")


def _taobao_bucketized_features() -> str:
    """The FG_NONE Taobao features of the bucketized examples: ids without expressions, price as 101 buckets, pid 2."""
    out = [_id_feature(n, None, r) for n, r in TAOBAO_USER + TAOBAO_ITEM]
    return "".join(out) + _id_feature("price", None, 101) + _id_feature("pid", None, 2)


def dbmtl_taobao_jrc() -> str:
    """examples/dbmtl_taobao_jrc.config: dbmtl_taobao on the bucketized FG_NONE features, with two-class towers trained
    by the JRC loss over sessions of `user_id` (cvr auc with 10000 thresholds)."""
    return (_header("taobao_multitask_sample_bucketized_train_jrc", "taobao_multitask_sample_bucketized_v1/ds=20170513",
                    "taobao/dbmtl_jrc", "FG_NONE", ["clk", "buy"], None, quota=False)
            + _taobao_bucketized_features()
            + "model_config {\n" + _group("all", TAOBAO_MMOE_ORDER, "DEEP")
            + "    dbmtl {\n" + _mlp("bottom_mlp", [512], "        ")
            + _dbmtl_towers(10000, 'jrc_loss {\n                    session_name: "user_id"\n                }',
                            "            num_class: 2\n") + "    }\n}\n")


def dbmtl_taobao_seq() -> str:
    """examples/dbmtl_taobao_seq.config: dbmtl_taobao on the bucketized FG_NONE features plus click_50_seq (adgroup_id,
    cate_id, brand; up to 100), whose sequence group sits inside the DEEP group `all` with a DIN encoder (attention MLP
    32-8); BCE towers, cvr auc with 10000 thresholds."""
    seq_feats = "".join(
        "        features {\n            id_feature {\n"
        f'                feature_name: "{n}"\n                num_buckets: {r}\n                embedding_dim: 16\n'
        "            }\n        }\n" for n, r in [("adgroup_id", 846812), ("cate_id", 12961), ("brand", 461498)])
    seq = ('feature_configs {\n    sequence_feature {\n        sequence_name: "click_50_seq",\n'
           '        sequence_length: 100\n        sequence_delim: "|"\n' + seq_feats + "    }\n}\n")
    names = "".join(f'            feature_names: "{f}"\n' for f in
                    ["adgroup_id", "cate_id", "brand", "click_50_seq__adgroup_id", "click_50_seq__cate_id",
                     "click_50_seq__brand"])
    group = _group("all", TAOBAO_MMOE_ORDER, "DEEP")
    group = group[:group.rindex("    }\n")] + (
        '        sequence_groups {\n            group_name: "click_50_seq"\n' + names + "        }\n"
        "        sequence_encoders {\n            din_encoder {\n" + _mlp("attn_mlp", [32, 8], "                ")
        + "            }\n        }\n    }\n")
    return (_header("taobao_multitask_sample_bucketized_train", "taobao_multitask_sample_bucketized_v1/ds=20170513",
                    "taobao/dbmtl_seq", "FG_NONE", ["clk", "buy"], None, quota=False)
            + _taobao_bucketized_features() + seq
            + "model_config {\n" + group
            + "    dbmtl {\n" + _mlp("bottom_mlp", [512], "        ")
            + _dbmtl_towers(10000, "binary_cross_entropy {}") + "    }\n}\n")


def dbmtl_taobao_seq_encoders() -> str:
    """dbmtl_taobao_seq with two more encoders on click_50_seq beside its DIN encoder: `self_attention_encoder {}` (512
    dims, 8 heads) and `pooling_encoder { pooling_type: "mean" }`.  The edit: the reference ships no example with these
    encoders in a DEEP group."""
    extra = ("        sequence_encoders {\n            self_attention_encoder {\n            }\n        }\n"
             "        sequence_encoders {\n            pooling_encoder {\n"
             '                pooling_type: "mean"\n            }\n        }\n')
    text = dbmtl_taobao_seq()
    end = text.index("    dbmtl {\n")
    head = text[:end]
    close = head.rindex("    }\n")
    return (head[:close] + extra + head[close:] + text[end:]).replace('dbmtl_seq"', 'dbmtl_seq_encoders"')


def rocket_launching_criteo() -> str:
    """examples/rocket_launching_criteo.config: dlrm_criteo's features in one DEEP group `deep` (13 raw + 26 id(D=16),
    429 wide); rocket_launching{booster 256-128-64-32, light 96-64-32, feature_based_distillation}; a two-class head
    with softmax cross-entropy."""
    ints = [f"int_{i}" for i in range(13)]
    cats = [f"cat_{i}" for i in range(26)]
    return (_header("criteo_terabyte_train_hashed_v1", "criteo_terabyte_val_test_hashed_v1", "rocket_launch_criteo",
                    "FG_DAG", ["label"], 100)
            + _criteo_features(True)
            + "model_config {\n" + _group("deep", ints + cats, "DEEP")
            + "    rocket_launching {\n" + _mlp("booster_mlp", [256, 128, 64, 32], "        ")
            + _mlp("light_mlp", [96, 64, 32], "        ") + "        feature_based_distillation: true\n    }\n"
            "    num_class: 2\n"
            "    metrics {\n        auc {}\n    }\n    losses {\n        softmax_cross_entropy {}\n    }\n}\n")


def tdm_taobao() -> str:
    """examples/tdm_taobao.config: the Taobao user and item id features (D=16) with the item tables shared by name
    (item_emb, cate_emb, brand_emb) and the three click_50_seq__{adgroup_id,cate_id,brand} sequence id features (up to
    50) of one behaviour list; a SEQUENCE group `seq` (the three sequences, queried by adgroup_id, cate_id, brand),
    DEEP groups `user` and `item`; tdm{multiwindow_din{windows 1,1,1,2,2,2,5,6,10,20, attn_mlp 36 PReLU}, final
    256-128-64-32 with BN}; a two-class softmax cross-entropy head with auc.  data_config.tdm_sampler configures the
    reference's tree sampler (data pipeline, not the model)."""
    adam = "        adam_optimizer {\n            lr: 0.001\n        }\n        constant_learning_rate {\n        }\n"
    layers = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 17, 23, 30, 34, 82, 200]
    attrs = "".join(f'        attr_fields: "{a}"\n' for a in ["cate_id", "campaign_id", "customer", "brand", "price"])
    head = ('train_input_path: "data/taobao_data_recall_train_transformed/*.parquet"\n'
            'eval_input_path: "data/taobao_data_recall_eval_transformed/*.parquet"\n'
            'model_dir: "experiments/tdm_taobao"\n'
            "train_config {\n    sparse_optimizer {\n" + adam + "    }\n    dense_optimizer {\n" + adam + "    }\n"
            "    num_epochs: 2\n    log_step_count_steps: 1\n    save_checkpoints_steps: 100000\n}\n"
            "eval_config {\n}\n"
            "data_config {\n    batch_size: 32\n    dataset_type: ParquetDataset\n    fg_mode: FG_NONE\n"
            '    label_fields: "clk"\n    num_workers: 10\n    tdm_sampler {\n'
            "        item_input_path: 'data/init_tree/node_table.txt'\n"
            "        edge_input_path: 'data/init_tree/edge_table.txt'\n"
            "        predict_edge_input_path: 'data/init_tree/predict_edge_table.txt'\n" + attrs +
            '        item_id_field: "adgroup_id"\n'
            f"        layer_num_sample: [{', '.join(str(n) for n in layers)}]\n"
            "        attr_delimiter: ','\n    }\n}\n")
    user = [(n, r) for n, r in TAOBAO_USER]

    def named(name, side, rows, emb=None):
        f = _id_feature(name, side, rows)
        return f if emb is None else f.replace("        embedding_dim: 16\n",
                                               f'        embedding_dim: 16\n        embedding_name: "{emb}"\n')

    seqs = "".join(
        "feature_configs {\n    sequence_id_feature {\n"
        f'        feature_name: "click_50_seq__{n}"\n        sequence_length: 50\n        sequence_delim: ";"\n'
        f'        expression: "user:click_50_seq__{n}"\n        embedding_dim: 16\n        num_buckets: {r}\n'
        f'        embedding_name: "{e}"\n    }}\n}}\n'
        for n, r, e in [("adgroup_id", 1895387, "item_emb"), ("cate_id", 12961, "cate_emb"),
                        ("brand", 461498, "brand_emb")])
    feats = ("".join(named(n, "user", r) for n, r in user) + seqs
             + named("adgroup_id", "item", 1895387, "item_emb") + named("cate_id", "item", 12961, "cate_emb")
             + named("campaign_id", "item", 423438) + named("customer", "item", 255877)
             + named("brand", "item", 461498, "brand_emb") + named("price", "item", 100)
             + _id_feature("pid", "context", 20, field="hash_bucket_size"))
    seq_names = ["click_50_seq__adgroup_id", "click_50_seq__cate_id", "click_50_seq__brand", "adgroup_id", "cate_id",
                 "brand"]
    return (head + feats + "model_config {\n" + _group("seq", seq_names, "SEQUENCE")
            + _group("user", [n for n, _ in user] + ["pid"], "DEEP")
            + _group("item", ["campaign_id", "customer", "price"], "DEEP")
            + "    tdm {\n        multiwindow_din {\n            windows_len: [1, 1, 1, 2, 2, 2, 5, 6, 10, 20]\n"
            + _mlp("attn_mlp", [36], "            ").replace("hidden_units: [36]\n",
                                                             "hidden_units: [36]\n                activation: 'nn.PReLU'\n")
            + "        }\n" + _mlp("final", [256, 128, 64, 32], "        ").replace(
                "hidden_units: [256, 128, 64, 32]\n", "hidden_units: [256, 128, 64, 32]\n            use_bn: true\n")
            + "    }\n    num_class: 2\n"
            "    metrics {\n        auc {}\n    }\n    losses {\n        softmax_cross_entropy {}\n    }\n}\n")


def dcn_v2_taobao() -> str:
    """examples/multi_tower_taobao.config with ONE edit: its model_config replaced by the dcn_v2 example of the
    reference's docs/source/models/dcn_v2.md (the reference ships no DCN-v2 example file).  The 16 Taobao features
    (16 wide each, D = 256) in one DEEP group `features`; backbone 512-256-128, so the cross network runs at D = 128
    with cross_num 2 and low_rank 32; deep 512-256 on the raw group; final 128-32; auc and binary cross-entropy."""
    return (_header("taobao_multitask_sample_v1_train", "taobao_multitask_sample_v1/ds=20170513",
                    "multi_tower_taobao", "FG_DAG", ["clk"], None, quota=False)
            + _taobao_features()
            + "model_config {\n" + _group("features", TAOBAO_MMOE_ORDER, "DEEP")
            + "    dcn_v2 {\n" + _mlp("backbone", [512, 256, 128], "        ")
            + "        cross {\n            cross_num: 2\n            low_rank: 32\n        }\n"
            + _mlp("deep", [512, 256], "        ") + _mlp("final", [128, 32], "        ")
            + "    }\n    num_class: 1\n"
            "    metrics {\n        auc {}\n    }\n    losses {\n        binary_cross_entropy {}\n    }\n}\n")


GENERATORS = {"dlrm_criteo": dlrm_criteo, "deepfm_criteo": deepfm_criteo, "mmoe_taobao": mmoe_taobao,
              "multi_tower_din_taobao": multi_tower_din_taobao, "masknet_criteo": masknet_criteo,
              "ple_taobao": ple_taobao, "pepnet_taobao": pepnet_taobao, "dbmtl_taobao": dbmtl_taobao,
              "dbmtl_taobao_jrc": dbmtl_taobao_jrc, "dbmtl_taobao_seq": dbmtl_taobao_seq,
              "rocket_launching_criteo": rocket_launching_criteo, "tdm_taobao": tdm_taobao}
# built-in configs that differ from their reference example by a documented edit (each generator's docstring names it),
# so they are not in GENERATORS, whose every entry parses to the same tree as the reference's file
EDITED_GENERATORS = {"wukong_criteo": wukong_criteo, "dcn_v2_taobao": dcn_v2_taobao,
                     "dbmtl_taobao_seq_encoders": dbmtl_taobao_seq_encoders}
# every built-in config by name (engine.Pipeline resolves names here)
BUILTINS = {**GENERATORS, **EDITED_GENERATORS}


def write_config(name: str, path: str) -> str:
    with open(path, "w") as fh:
        fh.write(BUILTINS[name]())
    return path
