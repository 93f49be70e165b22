"""In-tree build of libpvb200.so (sm_90a only) with plain nvcc.

The built library is git-ignored; build() makes it from the sources.  nvcc cross-compiles without a GPU,
so the library can be built on a machine that has none.
"""
import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_DIR = os.path.join(_HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libpvb200.so")
SOURCES = ["pv_api.cu", "pv_transform.cu", "pv_augment.cu", "pv_roi.cu", "pv_simt.cu", "pv_igemm.cu", "pv_igemm_gather.cu", "pv_dwconv.cu", "pv_dwlane.cu", "pv_dwplane.cu","pv_fastblock.cu", "pv_stem.cu", "pv_stem_stream.cu", "pv_attention.cu", "pv_attention_mma.cu", "pv_attention_wgmma.cu", "pv_attention_wide.cu", "pv_mix.cu", "pv_masked.cu", "pv_lstm.cu", "pv_boxes.cu", "pv_boxes_ragged.cu", "pv_contrastive.cu", "pv_colorjitter.cu", "pv_bank.cu", "pv_jpeg.cu"]
ARCH = "arch=compute_90a,code=sm_90a"
NVCC_FLAGS = [
    "-gencode", ARCH, "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-diag-suppress", "550",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(_HERE, "..", "include", "pv_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    """Compile every CUDA source (one object per .cu, in parallel, only the stale ones) and link lib/libpvb200.so.
    Returns the library path."""
    if not force and not needs_build():
        return LIB_PATH
    nvcc = _nvcc()
    if nvcc is None:
        if os.path.exists(LIB_PATH):   # a machine without nvcc: keep the library built earlier
            return LIB_PATH
        raise RuntimeError("nvcc not found and no prebuilt libpvb200.so present")
    from concurrent.futures import ThreadPoolExecutor
    obj_dir = os.path.join(LIB_DIR, "obj")
    os.makedirs(obj_dir, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if not f.endswith(".cu")]
    headers.append(os.path.join(_HERE, "..", "include", "pv_b200.h"))
    t_hdr = max(os.path.getmtime(h) for h in headers if os.path.exists(h))
    flags = [f for f in NVCC_FLAGS if f != "-shared"]

    def compile_one(src):
        obj = os.path.join(obj_dir, src[:-3] + ".o")
        path = os.path.join(CSRC, src)
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(t_hdr, os.path.getmtime(path)):
            return obj, None
        tmp = obj + ".tmp.%d" % os.getpid()
        res = subprocess.run([nvcc] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", tmp, path],
                             capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n" % src + res.stdout + res.stderr)
        os.replace(tmp, obj)
        return obj, res.stderr

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 4)) as ex:
        results = list(ex.map(compile_one, SOURCES))
    if verbose:
        for _, err in results:
            if err:
                print(err)
    tmp = LIB_PATH + ".tmp.%d" % os.getpid()
    res = subprocess.run([nvcc, "-shared", "-gencode", ARCH, "-o", tmp] + [o for o, _ in results],
                         capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc link failed:\n" + res.stdout + res.stderr)
    os.replace(tmp, LIB_PATH)
    return LIB_PATH


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
