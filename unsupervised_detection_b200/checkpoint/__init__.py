"""Checkpoint I/O: TF V2 tensor-bundle files (the reference's tf.train.Saver format) and the TF variable-name map."""
from .tf_bundle import (read_bundle, write_bundle, list_variables, is_bundle, latest_checkpoint,  # noqa: F401
                        update_checkpoint_state, read_checkpoint_state)
from .tf_names import ema_name, export_params, import_params, normalize_prefix, to_tf_name  # noqa: F401
