"""Boundary test (SURVEY §8b recipe): what the reference's UNCHANGED callers — `trainer/trainer.py:Trainer`,
`trainer/base_trainer.py` checkpointing and resume, `util/utils.py:initialize_config / load_checkpoint` and the `enhancement.py`
script — computed with the drop-in (or with the reference module, where the drop-in must reproduce it), recorded as golden data
by `oracle/gen_golden_boundary.py` from a checkout of the reference. Here the drop-in goes through the same calls those callers
make (restated from the cited lines) and must reproduce the recorded parameters, losses and outputs. There is no GPU here, so
  * the training loop runs the drop-in with ``train_backend="torch"`` (the composite that runs on CPU; the native kernels are
    compared with it and with the float64 goldens in tests/test_train_gpu.py);
  * for the enhancement loop the ONE native call (``Model._forward_native``) is replaced by the torch restatement of the same
    formulas — everything around it (strict checkpoint load, `.to()/.eval()`, the [1,1,16384] chunk calls, `.detach().cpu()`,
    trimming) is the real shim. The native forward's numerics are the GPU parity tests' job."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import boundary_common as bc


@pytest.fixture(scope="module")
def gold(golden_dir):
    def load(name):
        return np.load(os.path.join(golden_dir, name))
    return load


def initialize_config(stanza):
    """util/utils.py:initialize_config: the class named by "module" / "main", constructed with "args" """
    return getattr(importlib.import_module(stanza["module"]), stanza["main"])(**stanza["args"])


def golden_state(g, prefix):
    return {k.split(":", 1)[1]: torch.from_numpy(g[k]) for k in g.files if k.startswith(prefix + ":")}


def noise_driven(key):
    """Entries whose recorded value depends on the machine. The conv biases followed by BatchNorm have a true gradient of zero:
    backward yields rounding noise whose sign depends on the reduction order (CPU, thread count), and Adam turns it into a full
    +-lr step. The BatchNorm running statistics follow those biases."""
    return (key.endswith(".0.bias") and not key.startswith("out.")) or key.endswith(".running_mean") or key.endswith(".running_var")


def assert_state_matches(model, g, prefix, atol, steps, lr=1e-3, isolated=4):
    """Parameters and BatchNorm buffers against the recorded ones: the noise-driven entries within `steps` Adam steps of 2 lr;
    every other entry within atol, except at most `isolated` single entries whose own gradient happens to be at the rounding
    level (each still within the Adam bound)."""
    want = golden_state(g, prefix)
    got = model.state_dict()
    assert list(got) == list(want)
    bound = steps * 2 * lr * 1.05
    outliers = []
    for k, v in want.items():
        a, b = got[k].double(), v.double()
        if k.endswith("num_batches_tracked"):
            assert torch.equal(a, b), k
            continue
        d = (a - b).abs()
        assert float(d.max()) <= bound, (k, float(d.max()))
        if not noise_driven(k):
            outliers += [k] * int(d.gt(atol).sum())
    assert len(outliers) <= isolated, (prefix, outliers)


def make_trainer_parts(cfg):
    """train.py:29-35: model and loss from their config stanzas, Adam with the configured betas"""
    model = initialize_config(cfg["model"])
    optimizer = torch.optim.Adam(params=model.parameters(), lr=cfg["optimizer"]["lr"],
                                 betas=(cfg["optimizer"]["beta1"], cfg["optimizer"]["beta2"]))
    return model, optimizer


def train_epochs(model, optimizer, loader, first, last, ck):
    """base_trainer.py:189-212 + trainer.py:27-42 (train mode, one optimizer step per batch) and the checkpoint files of
    base_trainer.py:83-127 (latest_model.tar with epoch / best_score / optimizer / model, model_<epoch>.pth)"""
    for epoch in range(first, last + 1):
        model.train()
        for batch in loader:
            bc.adam_step(model, optimizer, batch)
        module = model.module if isinstance(model, torch.nn.DataParallel) else model
        torch.save({"epoch": epoch, "best_score": -np.inf, "optimizer": optimizer.state_dict(), "model": module.cpu().state_dict()},
                   os.path.join(ck, "latest_model.tar"))
        torch.save(module.state_dict(), os.path.join(ck, f"model_{str(epoch).zfill(4)}.pth"))


def test_unchanged_trainer_trains_checkpoints_and_resumes_the_dropin(gold, tmp_path):
    g = gold("boundary_trainer.npz")
    ck = str(tmp_path)
    torch.manual_seed(bc.TRAINER_SEED)
    cfg = bc.train_config(tmp_path, 2)
    model, optimizer = make_trainer_parts(cfg)
    assert type(model).__module__ == bc.DROPIN
    before = [p.detach().clone() for p in model.parameters()]
    train_epochs(model, optimizer, bc.synthetic_loader(), 1, 2, ck)
    assert any(not torch.equal(a, b) for a, b in zip(before, model.parameters())), "optimizer never moved the parameters"
    # the reference Trainer, training the same drop-in from the same seed, reached these parameters (6 optimizer steps)
    assert_state_matches(model, g, "epoch2", 1e-6, steps=6)
    assert sorted(os.listdir(ck)) == [f for f in g["files"] if f != "model_0003.pth"]
    tar = torch.load(os.path.join(ck, "latest_model.tar"))
    assert sorted(tar) == list(g["tar_keys"]) and tar["epoch"] == int(g["tar_epoch"])

    # the checkpoint the reference wrote loads strictly into a fresh drop-in, which computes what the REFERENCE module computed
    # with it
    drop = importlib.import_module(bc.DROPIN).Model(bc.N, bc.CI, train_backend="torch")
    drop.load_state_dict(golden_state(g, "epoch2"))                                  # strict
    drop.eval()
    with torch.no_grad():
        assert np.abs(drop._forward_torch_reference_semantics(bc.probe_input()).numpy() - g["y_ref"]).max() <= 1e-6

    # resume (base_trainer.py:62-81): optimizer state (index-keyed) and model state come back, training continues at epoch 3
    model2, optimizer2 = make_trainer_parts(bc.train_config(tmp_path, 3))
    checkpoint = torch.load(os.path.join(ck, "latest_model.tar"))
    start_epoch = checkpoint["epoch"] + 1
    optimizer2.load_state_dict(checkpoint["optimizer"])
    model2.load_state_dict(checkpoint["model"])
    assert start_epoch == 3
    for a, b in zip(model2.state_dict().values(), tar["model"].values()):
        assert torch.equal(a, b)
    assert len(optimizer2.state_dict()["state"]) == len(list(model2.parameters()))
    train_epochs(model2, optimizer2, bc.synthetic_loader(), 3, 3, ck)
    assert_state_matches(model2, g, "epoch3", 1e-6, steps=9)

    # the nn.DataParallel branches of save / resume (base_trainer.py:76-77, 102-103): `.module` is the drop-in
    wrapped = torch.nn.DataParallel(model2)
    train_epochs(wrapped, optimizer2, [], 4, 4, ck)
    checkpoint = torch.load(os.path.join(ck, "latest_model.tar"))
    wrapped.module.load_state_dict(checkpoint["model"])
    assert checkpoint["epoch"] + 1 == 5 and type(wrapped.module).__module__ == bc.DROPIN


def test_adam_state_written_with_the_reference_model_continues_on_the_dropin(gold):
    """Adam's state is keyed by parameter INDEX (base_trainer.py:74,99): a run started with the reference module (its model and
    optimizer state after one step are recorded) and resumed with the drop-in must continue exactly as the reference did."""
    g = gold("boundary_adam.npz")
    drop = importlib.import_module(bc.DROPIN).Model(bc.N, bc.CI, train_backend="torch").train()
    drop.load_state_dict(golden_state(g, "model"))
    opt = torch.optim.Adam(drop.parameters(), lr=1e-3, betas=(0.9, 0.999))
    sd = opt.state_dict()
    sd["state"] = {i: {"step": torch.tensor(float(g["opt_step"])), "exp_avg": torch.from_numpy(g[f"exp_avg:{i}"]),
                       "exp_avg_sq": torch.from_numpy(g[f"exp_avg_sq:{i}"])} for i in range(len(sd["param_groups"][0]["params"]))}
    opt.load_state_dict(sd)
    got = bc.adam_step(drop, opt, bc.synthetic_loader()[1])
    want = float(g["loss"])
    assert abs(got - want) <= 1e-7 * abs(want)
    assert_state_matches(drop, g, "after", 1e-7, steps=1)


def test_unchanged_enhancement_script_runs_the_dropin(gold, tmp_path, monkeypatch):
    """enhancement.py:36-80 (strict checkpoint load of the "args": {} model, chunk loop, trimming) with the drop-in; the same
    checkpoint and clips through the unchanged script with the reference module gave the recorded wav outputs."""
    g = gold("boundary_enhance.npz")
    drop_mod = importlib.import_module(bc.DROPIN)
    monkeypatch.setattr(drop_mod.Model, "_forward_native", lambda self, x: self._forward_torch_reference_semantics(x).detach())
    ckpt = tmp_path / "model_0001.pth"
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in bc.enhance_state().items()}, ckpt)
    model = initialize_config({"module": bc.DROPIN, "main": "Model", "args": {}})
    model.load_state_dict(torch.load(ckpt, map_location="cpu"))                      # strict
    model.to(torch.device("cpu"))
    model.eval()
    sample_length = 16384
    clips = bc.enhance_clips()
    assert sorted(clips) == sorted(g.files) == ["a", "b"]
    for name, clip in clips.items():
        mixture = torch.from_numpy(clip).reshape(1, 1, -1)
        padded_length = 0
        if mixture.size(-1) % sample_length != 0:
            padded_length = sample_length - (mixture.size(-1) % sample_length)
            mixture = torch.cat([mixture, torch.zeros(1, 1, padded_length)], dim=-1)
        enhanced = torch.cat([model(chunk).detach().cpu() for chunk in torch.split(mixture, sample_length, dim=-1)], dim=-1)
        enhanced = enhanced if padded_length == 0 else enhanced[:, :, :-padded_length]
        enhanced = enhanced.reshape(-1).numpy()
        assert enhanced.shape == g[name].shape == clip.shape
        assert np.abs(enhanced - g[name]).max() <= 1e-6, name


def test_dataset_plugin_is_selected_by_the_config_stanza_and_feeds_the_unchanged_trainer(gold, tmp_path):
    """config/train/train.json:37-47 with only the "module" string changed: initialize_config builds the drop-in Dataset, a stock
    DataLoader batches it (train.py:15-27), and one epoch of the trainer's loop on those batches reaches the parameters the
    reference Trainer reached."""
    from torch.utils.data import DataLoader
    g = gold("boundary_dataset_plugin.npz")
    listing = bc.write_plugin_pairs(str(tmp_path))
    dataset = initialize_config(bc.plugin_stanza(listing))                           # train.py:15
    assert type(dataset).__module__ == "wave_u_net_for_speech_enhancement_b200.dataset" and len(dataset) == 6
    np.random.seed(0)
    batches = list(DataLoader(dataset=dataset, batch_size=3, num_workers=0, shuffle=False))
    assert len(batches) == 2 and batches[0][0].shape == (3, 1, 64) and batches[0][0].dtype == torch.float32
    assert [n for b in batches for n in b[2]] == list(g["names"])
    torch.manual_seed(bc.PLUGIN_SEED)
    model, optimizer = make_trainer_parts(bc.train_config(tmp_path, 1))
    before = [p.detach().clone() for p in model.parameters()]
    ck = tmp_path / "ck"
    ck.mkdir()
    train_epochs(model, optimizer, batches, 1, 1, str(ck))
    assert any(not torch.equal(a, b) for a, b in zip(before, model.parameters()))
    assert_state_matches(model, g, "epoch1", 1e-6, steps=2)
