"""Record tests/golden/forward_io_sass.json: per kernel of the inference units, a sha256 of its SASS and its resource usage.

The inference kernels that read the network input or write its output take the I/O element type as a template argument (float,
__half or __nv_bfloat16), so that a half model reads and writes 16-bit samples. Their float forms must compile to the machine
code they compiled to before that argument existed, and so must every other kernel of these units. The golden is therefore
recorded from the commit before the change:
    git archive <commit> | tar -x -C /tmp/parent
    python tools/gen_forward_io_sass_golden.py --csrc /tmp/parent/wave_u_net_for_speech_enhancement_b200/csrc
and tests/test_half_io_cpu.py computes the same record for the tree. A kernel's key is its unit and its demangled name with the
template arguments and without the parameter list; a trailing `float` I/O argument is dropped from the key, and the 16-bit I/O
forms (new kernels) are left out of the record. Digests and resource lines are computed as in gen_train_tc_sass_golden.py."""
import argparse
import json
import os
import re
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gen_train_tc_sass_golden as sass  # noqa: E402

ROOT = sass.ROOT
UNITS = ["wunet_fp32.cu", "wunet_tc.cu", "wunet_tc_f16.cu", "wunet_tc_wide.cu"]
IO16 = ("__half", "__nv_bfloat16")


def kernel_key(unit, demangled):
    """unit:name<template arguments> with a float I/O argument dropped, or None for a 16-bit I/O form"""
    s = demangled[5:] if demangled.startswith("void ") else demangled
    cut = s.find(">(")
    name = s[:cut + 1] if cut >= 0 else s[:s.index("(")]
    if cut >= 0:
        targs = name[name.index("<"):]
        if any(t in targs for t in IO16):
            return None
        name = name.replace("<float>", "").replace(", float>", ">")
    return unit + ":" + name


def record(nvcc, csrc, tmp, units=UNITS):
    rec = {}
    for u in units:
        obj = os.path.join(tmp, u.replace(".cu", ".o"))
        sass.compile_unit(nvcc, os.path.join(csrc, u), obj)
        k = sass.kernels(nvcc, obj, key_of=lambda d, u=u: kernel_key(u, d) or "io16:" + d)
        rec.update({key: v for key, v in k.items() if not key.startswith("io16:")})
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--csrc", required=True, help="csrc directory of the tree to record")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "forward_io_sass.json"))
    a = ap.parse_args()
    nvcc = sass.nvcc_path()
    with tempfile.TemporaryDirectory() as tmp:
        rec = record(nvcc, a.csrc, tmp)
    g = {"note": "per kernel of the inference units: sha256 of the whitespace-normalised instruction and encoding lines of "
                 "cuobjdump -sass, and the cuobjdump -res-usage line (tools/gen_forward_io_sass_golden.py)",
         "nvcc": sass.nvcc_release(nvcc), "flags": sass.NVCC_FLAGS,
         "kernels": {k: {"sass": v["sass"], "res": v["res"]} for k, v in sorted(rec.items())}}
    with open(a.out, "w") as f:
        json.dump(g, f, indent=1)
        f.write("\n")
    print("wrote", len(g["kernels"]), "kernels to", a.out)


if __name__ == "__main__":
    main()
