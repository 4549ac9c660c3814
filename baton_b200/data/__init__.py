"""Synthetic private shards (there is no dataset access on the target box)."""
from .synthetic import (LINEAR_TRUTH, ShardSpec, class_means, client_holdout_image_shard, dirichlet_label_shards,
                        holdout_image_shard, holdout_token_shard, image_shard, iid_label_shards, label_skew_shards,
                        linear_regression_shard, token_shard)

__all__ = ["LINEAR_TRUTH", "ShardSpec", "linear_regression_shard", "image_shard", "token_shard",
           "iid_label_shards", "label_skew_shards", "dirichlet_label_shards",
           "holdout_image_shard", "holdout_token_shard", "class_means", "client_holdout_image_shard"]
