"""The RocketLaunching cases of tests/golden/ref_rocket.npz (made by tests/golden/make_rocket_golden.py from the
reference's own RocketLaunching): each case's model sub-message, and the same case as a pipeline config for this
repo's model.  The group input is D = 24 wide (three 8-wide id features here; the seeded input is fed in place of the
embedding lookup), B = 16 samples."""

D, B = 24, 16
SIMILARITY = {"COSINE": 0, "INNER_PRODUCT": 1, "EUCLID": 2}          # tzrec/protos/simi.proto

# tag -> (rocket_launching sub-message, num_class, label_smoothing, zero light row)
CASES = {
    "example": (dict(booster_mlp=[256, 128, 64, 32], light_mlp=[96, 64, 32], feature_based_distillation=True),
                2, 0.0, False),
    "share_mlp": (dict(share_mlp=[32], booster_mlp=[32, 16, 8], light_mlp=[16, 16, 8],
                       feature_based_distillation=True), 2, 0.0, False),
    "distill_off": (dict(booster_mlp=[32, 16], light_mlp=[12, 20]), 2, 0.0, False),
    "euclid": (dict(booster_mlp=[32, 16, 8], light_mlp=[16, 8], feature_based_distillation=True,
                    feature_distillation_function="EUCLID"), 2, 0.0, False),
    "inner_product": (dict(booster_mlp=[32, 16, 8], light_mlp=[16, 8], feature_based_distillation=True,
                           feature_distillation_function="INNER_PRODUCT"), 2, 0.0, False),
    "three_class_eps": (dict(booster_mlp=[32, 16], light_mlp=[16], feature_based_distillation=True), 3, 0.1, False),
    "zero_light_row": (dict(booster_mlp=[32, 16, 8], light_mlp=[16, 8], feature_based_distillation=True),
                       2, 0.0, True),
}


def config_text(tag):
    """The case as a pipeline config: three 8-wide id features in group `deep` (width D)."""
    sub, C, eps, _ = CASES[tag]
    body = ""
    for k in ("share_mlp", "booster_mlp", "light_mlp"):
        if k in sub:
            body += f"    {k} {{ hidden_units: [{', '.join(str(u) for u in sub[k])}] }}\n"
    if sub.get("feature_based_distillation"):
        body += "    feature_based_distillation: true\n"
    if "feature_distillation_function" in sub:
        body += f"    feature_distillation_function: {sub['feature_distillation_function']}\n"
    feats = "".join(f'feature_configs {{ id_feature {{ feature_name: "f{i}" num_buckets: 20 embedding_dim: 8 }} }}\n'
                    for i in range(3))
    return (feats + 'model_config {\n  feature_groups { group_name: "deep" feature_names: ["f0", "f1", "f2"] '
            "group_type: DEEP }\n  rocket_launching {\n" + body + "  }\n"
            f"  num_class: {C}\n  metrics {{ auc {{}} }}\n"
            f"  losses {{ softmax_cross_entropy {{ label_smoothing: {eps} }} }}\n}}\n")
