"""Record tests/golden/train_tc_sass.json: per kernel of the tensor-core training convolutions, a sha256 of its SASS and its
resource usage, keyed by what the kernel computes rather than by its mangled name.

The bf16 and tf32 training convolutions were once two units and are now one, templated on the operand type; the merge must
leave every kernel's machine code as it was. The golden is therefore recorded from the commit before the merge:
    git archive <commit> | tar -x -C /tmp/parent
    python tools/gen_train_tc_sass_golden.py --csrc /tmp/parent/wave_u_net_for_speech_enhancement_b200/csrc
(by default every wunet_train_t*.cu unit of the tree: there, the bf16 and the tf32 one), and
tests/test_train_tc_unit_cpu.py computes the same record for the one unit of the tree. A kernel's key is pass/precision/KS/MODE/NT
for the convolutions (conv/bf16/15/0/1), pass/precision/KS/MODE/SLICES for the weight gradients (wgrad/tf32/5/2/1) and
pass/precision for the packing (pack/bf16). The digest covers the whitespace-normalised instruction and encoding lines of
`cuobjdump -sass`; the resource line is `cuobjdump -res-usage`'s (registers, stack, shared, local, constant).
`--dump DIR` also writes each kernel's normalised SASS there, for a diff against the same dump of another tree."""
import argparse
import glob
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DWUNET_BUILD"]


def nvcc_path():
    sys.path.insert(0, ROOT)
    from wave_u_net_for_speech_enhancement_b200 import build
    return build.nvcc_path()


def nvcc_release(nvcc):
    m = re.search(r"release \d+\.\d+, V([\d.]+)", subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout)
    return m and m.group(1)


def compile_unit(nvcc, src, obj, extra=()):
    """nvcc -c src -o obj with the flags the golden was recorded with; returns the compiler's output"""
    r = subprocess.run([nvcc] + NVCC_FLAGS + list(extra) + ["-c", src, "-o", obj], capture_output=True, text=True)
    log = r.stdout + r.stderr
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed on {src}:\n{log[-4000:]}")
    return log


def kernel_key(demangled):
    """the key of one kernel from its demangled name: the pass from the name, the precision from the name or the operand traits
    (tf32 where either says so, bf16 otherwise), then the integer and bool template arguments in order"""
    m = re.search(r"(train_\w+)_kernel(?:<(.*?)>)?\(", demangled)
    if m is None:
        raise ValueError(f"not a training tensor-core kernel: {demangled}")
    name, targs = m.group(1), m.group(2) or ""
    kind = next(k for k in ("conv", "wgrad", "pack") if k in name)
    prec = "tf32" if "tf32" in (name + targs).lower() else "bf16"
    return "/".join([kind, prec] + re.findall(r"\((?:int|bool)\)(\d+)", targs))


def demangle(nvcc, names):
    out = subprocess.run([os.path.join(os.path.dirname(nvcc), "cu++filt")], input="\n".join(names) + "\n", capture_output=True,
                         text=True, check=True).stdout.splitlines()
    return dict(zip(names, out))


def keys_of(nvcc, names):
    """{mangled name: key}"""
    return {n: kernel_key(d) for n, d in demangle(nvcc, names).items()}


def kernels(nvcc, obj, key_of=None):
    """{key: {"sass": sha256 of the normalised instruction lines, "res": resource line}} of every kernel in the object, plus the
    normalised SASS itself under "lines" (not recorded in the golden). key_of: demangled name -> key (default: kernel_key)"""
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    res = subprocess.run([cuobjdump, "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"\n\s*Function : (\S+)\n", sass)
    bodies = dict(zip(parts[1::2], parts[2::2]))
    usage = dict(re.findall(r"\n\s*Function (\S+):\n\s*(.+)", res))
    assert bodies.keys() == usage.keys(), (sorted(bodies), sorted(usage))
    keys = keys_of(nvcc, list(bodies)) if key_of is None else {n: key_of(d) for n, d in demangle(nvcc, list(bodies)).items()}
    assert len(set(keys.values())) == len(keys), "two kernels share a key"
    out = {}
    for name, body in bodies.items():
        lines = [" ".join(line.split()) for line in body.splitlines() if re.match(r"\s*/\*([0-9a-f]{4}\*/| 0x[0-9a-f]{16} \*/)", line)]
        out[keys[name]] = {"sass": hashlib.sha256("\n".join(lines).encode()).hexdigest(), "res": " ".join(usage[name].split()),
                           "lines": lines}
    return out


def record(nvcc, csrc, sources, tmp):
    rec = {}
    for s in sources:
        obj = os.path.join(tmp, s.replace(".cu", ".o"))
        compile_unit(nvcc, os.path.join(csrc, s), obj)
        k = kernels(nvcc, obj)
        assert not rec.keys() & k.keys(), f"{s} repeats kernels {sorted(rec.keys() & k.keys())}"
        rec.update(k)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--csrc", required=True, help="csrc directory of the tree to record")
    ap.add_argument("sources", nargs="*", help="units holding the kernels (default: every wunet_train_t*.cu in --csrc)")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "train_tc_sass.json"))
    ap.add_argument("--dump", default=None, help="also write each kernel's normalised SASS to this directory")
    a = ap.parse_args()
    nvcc = nvcc_path()
    sources = a.sources or sorted(os.path.basename(p) for p in glob.glob(os.path.join(a.csrc, "wunet_train_t*.cu")))
    with tempfile.TemporaryDirectory() as tmp:
        rec = record(nvcc, a.csrc, sources, tmp)
    if a.dump:
        os.makedirs(a.dump, exist_ok=True)
        for k, v in rec.items():
            with open(os.path.join(a.dump, k.replace("/", "_") + ".sass"), "w") as f:
                f.write("\n".join(v["lines"]) + "\n")
    g = {"note": "per kernel of the tensor-core training convolutions: sha256 of the whitespace-normalised instruction and encoding "
                 "lines of cuobjdump -sass, and the cuobjdump -res-usage line (tools/gen_train_tc_sass_golden.py)",
         "nvcc": nvcc_release(nvcc), "flags": NVCC_FLAGS,
         "kernels": {k: {"sass": v["sass"], "res": v["res"]} for k, v in sorted(rec.items())}}
    with open(a.out, "w") as f:
        json.dump(g, f, indent=1)
        f.write("\n")
    print("wrote", len(g["kernels"]), "kernels to", a.out)


if __name__ == "__main__":
    main()
