"""The ``derivative`` switch of a checkpoint (no GPU): ``load_model(path, derivative=...)`` in the reference
(``src/ViSNet/model/visnet.py:73-81``) takes the checkpoint's hyper-parameter unless a keyword overrides it.  Small
Lightning-style checkpoints are written with ``torch.save``; only the hyper-parameter handling is under test."""
import numpy as np
import pytest
import torch

from ai2bmd_b200.weights import load_checkpoint, load_state_dict, resolve_derivative

HP = dict(embedding_dimension=128, num_layers=6, num_heads=8, num_rbf=32, lmax=1, max_num_neighbors=32,
          vecnorm_type="max_min", rbf_type="expnorm", activation="silu", attn_activation="silu", cutoff=5.0,
          max_z=100, prior_model="Atomref", reduce_op="add")


def _ckpt(tmp_path, name, **hp):
    path = str(tmp_path / name)
    sd = {"model.representation_model.embedding.weight": torch.arange(6, dtype=torch.float32).reshape(2, 3),
          "model.std": torch.tensor(2.0)}
    torch.save({"hyper_parameters": {**HP, **hp}, "state_dict": sd}, path)
    return path


@pytest.mark.parametrize("value", [True, False])
def test_checkpoint_value_is_exposed(tmp_path, value):
    sd, derivative = load_checkpoint(_ckpt(tmp_path, "m.ckpt", derivative=value))
    assert derivative is value
    assert set(sd) == {"representation_model.embedding.weight", "std"}          # "model." stripped as before
    assert np.array_equal(sd["representation_model.embedding.weight"], np.arange(6, dtype=np.float32).reshape(2, 3))
    assert np.array_equal(load_state_dict(_ckpt(tmp_path, "n.ckpt", derivative=value))["std"], np.float32(2.0))


def test_checkpoint_without_the_key_counts_as_true(tmp_path):
    assert load_checkpoint(_ckpt(tmp_path, "m.ckpt"))[1] is True


def test_npz_counts_as_true(tmp_path):
    path = str(tmp_path / "w.npz")
    np.savez(path, a=np.ones(3, dtype=np.float32))
    sd, derivative = load_checkpoint(path)
    assert derivative is True and np.array_equal(sd["a"], np.ones(3, dtype=np.float32))


@pytest.mark.parametrize("ckpt,kw,want", [(True, None, True), (False, None, False), (True, False, False),
                                          (False, True, True), (True, True, True), (False, False, False)])
def test_keyword_overrides_the_checkpoint(ckpt, kw, want):
    assert resolve_derivative(ckpt, kw) is want


@pytest.mark.parametrize("key,value", [("num_layers", 4), ("embedding_dimension", 256), ("cutoff", 4.0),
                                       ("vecnorm_type", "none"), ("reduce_op", "mean"), ("derivative", "yes")])
def test_other_hyper_parameters_still_rejected(tmp_path, key, value):
    with pytest.raises(ValueError, match=key):
        load_checkpoint(_ckpt(tmp_path, "m.ckpt", **{key: value}))


def test_calculator_signature_takes_derivative():
    import inspect
    from ai2bmd_b200.calculator import ViSNetCalculator, ViSNetModel, get_visnet_model
    from ai2bmd_b200.engine import Engine
    assert inspect.signature(ViSNetCalculator).parameters["derivative"].default is None
    assert inspect.signature(get_visnet_model).parameters["derivative"].default is None
    assert inspect.signature(ViSNetModel).parameters["derivative"].default is True
    assert inspect.signature(Engine).parameters["derivative"].default is True
