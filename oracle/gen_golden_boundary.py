"""Record what the reference project's own callers compute around the drop-in, as golden data for tests/test_boundary_callers.py
and tests/test_dataset_cpu.py:

    python -m oracle.gen_golden_boundary /path/to/Wave-U-Net-for-Speech-Enhancement

The reference's UNCHANGED `Trainer` / `BaseTrainer` (training loop, checkpoint files, resume), `enhancement.py` and the
`Dataset` class of `dataset/waveform_dataset.py` are run here from a checkout of it; nothing of the reference is copied into
this repository. The packages it imports that are not needed for these paths (json5, librosa, pesq, pystoi, matplotlib) are
stubbed in `sys.modules`. Outputs (all under tests/golden/):
  boundary_trainer.npz        2 epochs of the reference Trainer on the drop-in, its checkpoint layout, a resumed 3rd epoch,
                              and the reference Model's output with the epoch-2 checkpoint
  boundary_adam.npz           one Adam step of the reference Model (model + index-keyed optimizer state) and the next step
  boundary_enhance.npz        enhancement.py's wav outputs for the reference Model on two clips
  boundary_dataset_plugin.npz 1 epoch of the reference Trainer on batches of the drop-in Dataset built by initialize_config
  dataset_reference_items.json digests of the reference Dataset's items (train and validation modes)
  reference_empty_batch.json  shape and dtype of the reference Model's eval forward on zero frames
"""
import copy
import importlib
import json
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import boundary_common as bc  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def stub_modules(wavs, written):
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    mod("json5", dumps=lambda o, **k: json.dumps(o, default=str), dump=lambda o, f, **k: json.dump(o, f, default=str),
        load=json.load, loads=json.loads)
    librosa = mod("librosa", load=lambda path, sr=None: (wavs[path].copy(), 16000) if path in wavs else bc.read_wav_f32(path),
                  stft=lambda y, **k: np.zeros((161, 4), np.complex64), magphase=lambda d: (np.abs(d), d),
                  amplitude_to_db=lambda m: m)
    librosa.output = mod("librosa.output", write_wav=lambda path, y, sr: written.__setitem__(path, np.asarray(y).copy()))
    librosa.display = mod("librosa.display", waveplot=lambda *a, **k: None, specshow=lambda *a, **k: None)
    mod("pesq", pesq=lambda sr, a, b, mode: 2.0)
    pystoi = mod("pystoi")
    pystoi.stoi = mod("pystoi.stoi", stoi=lambda a, b, sr, extended=False: 0.5)
    plt = mod("matplotlib.pyplot", switch_backend=lambda *a: None, subplots=lambda *a, **k: (None, None), tight_layout=lambda: None)
    mod("matplotlib", pyplot=plt)


def state_arrays(prefix, sd):
    return {f"{prefix}:{k}": v.detach().cpu().numpy() for k, v in sd.items()}


def build_trainer(cfg, resume, loader):
    utils = importlib.import_module("util.utils")
    model = utils.initialize_config(cfg["model"])
    optimizer = torch.optim.Adam(params=model.parameters(), lr=cfg["optimizer"]["lr"],
                                 betas=(cfg["optimizer"]["beta1"], cfg["optimizer"]["beta2"]))
    trainer_class = utils.initialize_config(cfg["trainer"], pass_args=False)
    return trainer_class(config=cfg, resume=resume, model=model, loss_function=utils.initialize_config(cfg["loss_function"]),
                         optimizer=optimizer, train_dataloader=loader, validation_dataloader=[])


def gen_trainer(tmp):
    torch.manual_seed(bc.TRAINER_SEED)
    t = build_trainer(bc.train_config(tmp, 2), False, bc.synthetic_loader())
    t.train()
    ck = os.path.join(tmp, "boundary", "checkpoints")
    tar = torch.load(os.path.join(ck, "latest_model.tar"))
    utils = importlib.import_module("util.utils")
    sd2 = utils.load_checkpoint(os.path.join(ck, "model_0002.pth"), torch.device("cpu"))
    ref = importlib.import_module("model.unet_basic").Model(n_layers=bc.N, channels_interval=bc.CI)
    ref.load_state_dict(sd2)
    ref.eval()
    with torch.no_grad():
        y_ref = ref(bc.probe_input()).numpy()
    t2 = build_trainer(bc.train_config(tmp, 3), True, bc.synthetic_loader())
    t2.train()
    sd3 = utils.load_checkpoint(os.path.join(ck, "model_0003.pth"), torch.device("cpu"))
    out = {"tar_keys": np.array(sorted(tar.keys())), "tar_epoch": np.int64(tar["epoch"]),
           "files": np.array(sorted(os.listdir(ck))), "y_ref": y_ref}
    out.update(state_arrays("epoch2", sd2))
    out.update(state_arrays("epoch3", sd3))
    np.savez_compressed(os.path.join(GOLD, "boundary_trainer.npz"), **out)


def gen_adam():
    ref_model_cls = importlib.import_module("model.unet_basic").Model
    torch.manual_seed(bc.ADAM_SEED)
    ref = ref_model_cls(n_layers=bc.N, channels_interval=bc.CI).train()
    opt = torch.optim.Adam(ref.parameters(), lr=1e-3, betas=(0.9, 0.999))
    batches = bc.synthetic_loader()
    bc.adam_step(ref, opt, batches[0])
    model_sd = {k: v.clone() for k, v in ref.state_dict().items()}
    opt_sd = copy.deepcopy(opt.state_dict())
    want = bc.adam_step(ref, opt, batches[1])
    out = {"loss": np.float64(want), "opt_step": np.float64(float(opt_sd["state"][0]["step"]))}
    out.update(state_arrays("model", model_sd))
    out.update(state_arrays("after", ref.state_dict()))
    for i, s in opt_sd["state"].items():
        out[f"exp_avg:{i}"] = s["exp_avg"].numpy()
        out[f"exp_avg_sq:{i}"] = s["exp_avg_sq"].numpy()
    np.savez_compressed(os.path.join(GOLD, "boundary_adam.npz"), **out)


def gen_enhance(ref_dir, tmp, wavs, written):
    ref = importlib.import_module("model.unet_basic").Model()
    ref.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in bc.enhance_state().items()})
    ckpt = os.path.join(tmp, "model_0001.pth")
    torch.save(ref.state_dict(), ckpt)
    listing = os.path.join(tmp, "list.txt")
    clips = bc.enhance_clips()
    paths = [os.path.join(tmp, f"{name}.wav") for name in clips]
    for p, name in zip(paths, clips):
        wavs[p] = clips[name]
    with open(listing, "w") as f:
        f.write("\n".join(paths) + "\n")
    cfg = {"model": {"module": "model.unet_basic", "main": "Model", "args": {}},
           "dataset": {"module": "dataset.waveform_dataset_enhancement", "main": "WaveformDataset",
                       "args": {"dataset": listing, "limit": None, "offset": 0, "sample_length": 16384}},
           "custom": {"sample_length": 16384}}
    cfg_path = os.path.join(tmp, "enh.json")
    with open(cfg_path, "w") as f:
        json.dump(cfg, f)
    out_dir = os.path.join(tmp, "enhanced")
    os.mkdir(out_dir)
    argv = sys.argv
    sys.argv = ["enhancement.py", "-C", cfg_path, "-D", "-1", "-O", out_dir, "-M", ckpt]
    written.clear()
    try:
        runpy.run_path(os.path.join(ref_dir, "enhancement.py"), run_name="__main__")
    finally:
        sys.argv = argv
    np.savez_compressed(os.path.join(GOLD, "boundary_enhance.npz"),
                        **{os.path.basename(k)[:-4]: v.astype(np.float32) for k, v in written.items()})


def gen_dataset_plugin(tmp):
    from torch.utils.data import DataLoader
    listing = bc.write_plugin_pairs(tmp)
    utils = importlib.import_module("util.utils")
    dataset = utils.initialize_config(bc.plugin_stanza(listing))
    np.random.seed(0)
    batches = list(DataLoader(dataset=dataset, batch_size=3, num_workers=0, shuffle=False))
    cfg = bc.train_config(tmp, 1)
    torch.manual_seed(bc.PLUGIN_SEED)
    t = build_trainer(cfg, False, batches)
    t.train()
    out = {"names": np.array([n for b in batches for n in b[2]])}
    out.update(state_arrays("epoch1", t.model.state_dict()))
    np.savez_compressed(os.path.join(GOLD, "boundary_dataset_plugin.npz"), **out)


def gen_dataset_items(tmp):
    lst, _ = bc.write_dataset_pairs(tmp)
    ref_ds = importlib.import_module("dataset.waveform_dataset")
    res = {}
    for mode in ("train", "validation"):
        r = ref_ds.Dataset(lst, sample_length=16384, mode=mode)
        np.random.seed(7)
        res[mode] = [bc.item_digest(r[i]) for i in range(len(r))]
    with open(os.path.join(GOLD, "dataset_reference_items.json"), "w") as f:
        json.dump(res, f, indent=1)


def gen_empty_batch():
    ref = importlib.import_module("model.unet_basic").Model(n_layers=bc.N, channels_interval=bc.CI).eval()
    with torch.no_grad():
        y = ref(torch.zeros(0, 1, 256))
    with open(os.path.join(GOLD, "reference_empty_batch.json"), "w") as f:
        json.dump({"input_shape": [0, 1, 256], "shape": list(y.shape), "dtype": str(y.dtype)}, f, indent=1)


def main():
    ref_dir = os.path.abspath(sys.argv[1])
    wavs, written = {}, {}
    stub_modules(wavs, written)
    sys.path.insert(0, ref_dir)
    with tempfile.TemporaryDirectory() as tmp:
        for sub in ("trainer", "adam", "enhance", "plugin", "items"):
            os.mkdir(os.path.join(tmp, sub))
        gen_trainer(os.path.join(tmp, "trainer"))
        gen_adam()
        gen_enhance(ref_dir, os.path.join(tmp, "enhance"), wavs, written)
        gen_dataset_plugin(os.path.join(tmp, "plugin"))
        gen_dataset_items(os.path.join(tmp, "items"))
        gen_empty_batch()
    print("wrote golden data under", GOLD)


if __name__ == "__main__":
    main()
