"""Inputs shared by oracle/gen_golden_boundary.py (which runs the reference project's own callers on them) and the tests that
check the drop-in against what those callers computed (tests/test_boundary_callers.py, tests/test_dataset_cpu.py). Everything
is generated from seeds, so both sides see the same data."""
import hashlib
import os

import numpy as np
import scipy.io.wavfile as wavfile
import torch

DROPIN = "wave_u_net_for_speech_enhancement_b200.unet_basic"
N, CI = 4, 8                       # architecture of the training-loop cases
TRAINER_SEED, ADAM_SEED, PLUGIN_SEED = 0, 1, 3


def train_config(root, epochs):
    """config/train/train.json with only the "model" stanza pointing at the drop-in (torch backend: runs on CPU)"""
    return {"seed": 0, "root_dir": str(root), "experiment_name": "boundary", "cudnn_deterministic": False,
            "trainer": {"module": "trainer.trainer", "main": "Trainer", "epochs": epochs, "save_checkpoint_interval": 1,
                        "validation": {"interval": 0, "find_max": True, "custom": {}}},
            "model": {"module": DROPIN, "main": "Model", "args": {"n_layers": N, "channels_interval": CI, "train_backend": "torch"}},
            "loss_function": {"module": "model.loss", "main": "mse_loss", "args": {}},
            "optimizer": {"lr": 0.001, "beta1": 0.9, "beta2": 0.999}}


def synthetic_loader(T=64, batches=3, B=4):
    """(mixture, clean, names) batches as train.py's DataLoader yields them"""
    g = torch.Generator().manual_seed(5)
    out = []
    for i in range(batches):
        clean = 0.1 * torch.randn(B, 1, T, generator=g)
        out.append((clean + 0.05 * torch.randn(B, 1, T, generator=g), clean, [f"f{i}_{j}" for j in range(B)]))
    return out


def probe_input():
    return torch.randn(2, 1, 64, generator=torch.Generator().manual_seed(11))


def adam_step(model, optimizer, batch):
    """one iteration of trainer/trainer.py:_train_epoch (zero_grad, forward, MSELoss(clean, enhanced), backward, step)"""
    mixture, clean, _ = batch
    optimizer.zero_grad()
    loss = torch.nn.MSELoss()(clean, model(mixture))
    loss.backward()
    optimizer.step()
    return float(loss.detach())


def enhance_state():
    """checkpoint of the enhancement case: the reference's default architecture, BatchNorm far from identity"""
    from oracle import wunet_oracle as wo
    return wo.make_state(12, 24, seed=2)


def enhance_clips():
    rng = np.random.default_rng(0)
    return {"a": (0.3 * rng.standard_normal(16384 + 4000)).astype(np.float32),    # padded to 2 chunks, trimmed
            "b": (0.3 * rng.standard_normal(16384)).astype(np.float32)}           # exactly one chunk


def write_plugin_pairs(root):
    """six short int16 (noisy, clean) wav pairs and their listing file (config/train/train.json "dataset" format)"""
    rng = np.random.default_rng(2)
    lines = []
    for i in range(6):
        n = 400 + 13 * i
        clean = rng.integers(-8000, 8000, n, dtype=np.int16)
        noisy = (clean + rng.integers(-900, 900, n)).astype(np.int16)
        wavfile.write(os.path.join(root, f"c{i}.wav"), 16000, clean)
        wavfile.write(os.path.join(root, f"n{i}.wav"), 16000, noisy)
        lines.append(f"{os.path.join(root, f'n{i}.wav')} {os.path.join(root, f'c{i}.wav')}")
    listing = os.path.join(root, "train.txt")
    with open(listing, "w") as f:
        f.write("\n".join(lines) + "\n")
    return listing


def plugin_stanza(listing):
    return {"module": "wave_u_net_for_speech_enhancement_b200.dataset", "main": "Dataset",
            "args": {"dataset": listing, "limit": None, "offset": 0, "sample_length": 64, "mode": "train"}}


def write_dataset_pairs(root, n_items=5, base_len=20000):
    """five (noisy, clean) int16 wav pairs of 20000+ samples and their listing file"""
    rng = np.random.default_rng(3)
    lines = []
    for i in range(n_items):
        n = base_len + 137 * i
        clean = rng.integers(-20000, 20000, n, dtype=np.int16)
        noisy = np.clip(clean.astype(np.int32) + rng.integers(-3000, 3000, n), -32768, 32767).astype(np.int16)
        pc, pn = os.path.join(root, f"clean_{i}.wav"), os.path.join(root, f"noisy_{i}.wav")
        wavfile.write(pc, 16000, clean)
        wavfile.write(pn, 16000, noisy)
        lines.append(f"{pn} {pc}")
    lst = os.path.join(root, "train.txt")
    with open(lst, "w") as f:
        f.write("\n".join(lines) + "\n")
    return lst, lines


def read_wav_f32(path):
    """what librosa.load(path, sr=None) returns for a mono int16 wav: float32 samples / 32768, the rate"""
    sr, a = wavfile.read(path)
    assert a.dtype == np.int16 and a.ndim == 1
    return a.astype(np.float32) / 32768.0, sr


def item_digest(item):
    """(mixture, clean, name) -> name, shapes and sha1 of the float32 bytes: exact equality without storing the audio"""
    mix, clean, name = item
    mix, clean = np.ascontiguousarray(mix, np.float32), np.ascontiguousarray(clean, np.float32)
    return {"name": name, "shape": list(mix.shape), "mix": hashlib.sha1(mix.tobytes()).hexdigest(),
            "clean": hashlib.sha1(clean.tobytes()).hexdigest()}
