"""compat/: the reference's import names over the engine (SURVEY.md 8b b1) -- host-only checks."""
import sys

from compat_helpers import COMPAT, write_experiment


def _import_compat():
    if COMPAT not in sys.path:
        sys.path.insert(0, COMPAT)
    import lvsr.config as C
    return C


def test_configuration_parent_changes_and_stages(tmp_path):
    """lvsr/config.py:9-92: parent links are merged recursively, command-line changes are parsed as YAML,
    stages are ordered by `number` and each stage is the base configuration plus its changes."""
    C = _import_compat()
    exp = write_experiment(tmp_path)
    cfg = C.Configuration(exp["child"], "$LVSR/lvsr/configs/schema.yaml",
                          [("net.conv_n", "6"), ("monitoring.search.beam_size", "5")])
    assert cfg["net"]["dims_bidir"] == [128] and cfg["net"]["conv_n"] == 6          # parent + change
    assert cfg["monitoring"]["search"]["beam_size"] == 5
    assert cfg["training"]["num_batches"] == 3 and cfg["training"]["gradient_threshold"] == 10.0
    assert cfg.multi_stage and list(cfg.ordered_stages) == ["pretraining", "main"]
    assert cfg.ordered_stages["pretraining"]["training"]["num_batches"] == 2
    assert cfg.ordered_stages["main"]["training"]["scale"] == 0.5 and "stages" not in cfg.ordered_stages["main"]
    # YAML python tags resolve to the engine's configuration tokens
    import _engine
    assert isinstance(cfg["net"]["post_merge_activation"], _engine.pkg.Maxout)
    assert cfg["net"]["post_merge_activation"].num_pieces == 2
    assert cfg["net"]["enc_transition"] is _engine.pkg.GatedRecurrent
    assert isinstance(cfg["initialization"]["/recognizer"]["rec_weights_init"], _engine.pkg.Orthogonal)


def test_dataset_batches_are_time_major_padded_and_masked(tmp_path):
    _import_compat()
    from lvsr.datasets import Data
    exp = write_experiment(tmp_path)
    data = Data(path=exp["npz"], batch_size=4, sort_k_batches=2)
    assert data.num_labels == 12 and data.eos_label == 11 and data.num_features == 40
    n = 0
    for b in data.batches("train"):
        T, B, F = b["recordings"].shape
        assert b["recordings_mask"].shape == (T, B) and b["labels"].shape[1] == B and b["labels"].dtype.kind == "i"
        last = b["labels_mask"].sum(axis=0).astype(int) - 1
        assert (b["labels"][last, range(B)] == data.eos_label).all()            # eos appended (datasets/__init__.py:267-270)
        assert (b["recordings"][b["recordings_mask"] == 0] == 0).all()
        n += B
    assert n == 10
