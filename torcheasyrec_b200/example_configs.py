"""Generators for the pipeline configs BASELINE.json names (text format, same message tree as the reference's
examples/{dlrm_criteo,deepfm_criteo,mmoe_taobao,multi_tower_din_taobao}.config).

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


GENERATORS = {"dlrm_criteo": dlrm_criteo, "deepfm_criteo": deepfm_criteo, "mmoe_taobao": mmoe_taobao,
              "multi_tower_din_taobao": multi_tower_din_taobao}


def write_config(name: str, path: str) -> str:
    with open(path, "w") as fh:
        fh.write(GENERATORS[name]())
    return path
