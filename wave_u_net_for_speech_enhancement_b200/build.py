"""In-tree build of libwunet_b200.so (nvcc, sm_90a only). `python -m wave_u_net_for_speech_enhancement_b200.build`"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libwunet_b200.so")
SOURCES = ["wunet_api.cu", "wunet_fp32.cu", "wunet_tc.cu", "wunet_train.cu"]
HEADERS = ["wunet_common.cuh", "wunet_tc.cuh", "wunet_train.cuh", os.path.join("..", "..", "include", "wunet_b200.h")]


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def is_stale() -> bool:
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def source_hash() -> str:
    """sha1 over the CUDA sources and headers (12 hex digits): compiled into wunet_version() so that recorded measurements can be
    matched to the binary they were taken from."""
    import hashlib
    h = hashlib.sha1()
    for s in SOURCES + HEADERS:
        with open(os.path.join(CSRC, s), "rb") as f:
            h.update(f.read())
    return h.hexdigest()[:12]


def build(force: bool = False, verbose: bool = False) -> str:
    out_so = os.environ.get("WUNET_SO_OUT") or SO            # development: variant builds next to the product library
    if out_so == SO and not force and not is_stale():
        return SO
    objs = []
    common = [nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-DWUNET_BUILD", f'-DWUNET_SRC_HASH="{source_hash()}"']
    if verbose:
        common += ["-Xptxas", "-v"]
    if os.environ.get("WUNET_TC_TRACE"):
        common += ["-DWUNET_TC_TRACE"]
    for macro in ("WUNET_WAIT_NS",):                  # development: mbarrier suspend-time hint (A/B builds)
        if os.environ.get(macro):
            common += [f"-D{macro}={int(os.environ[macro])}"]
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for s in SOURCES:
        o = os.path.join(HERE, "build", s.replace(".cu", ".o") if out_so == SO else os.path.basename(out_so) + "." + s.replace(".cu", ".o"))
        objs.append(o)
        cmd = common + ["-c", os.path.join(CSRC, s), "-o", o]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    link = [nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", out_so] + objs + ["-cudart", "static"]
    subprocess.check_call(link)
    return out_so


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
