"""In-tree build of libmyo_b200.so (H100, sm_90a only)."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "myo_b200.cu")
DEPS = [SRC, os.path.join(HERE, "csrc", "myo_device.cuh"), os.path.join(HERE, "csrc", "myo_solver.cuh"), os.path.join(HERE, "csrc", "myo_layout.cuh"),
        os.path.join(HERE, "..", "include", "myo_b200.h"), os.path.join(HERE, "..", "include", "myo_blob_layout.h"),
        os.path.join(HERE, "..", "include", "myo_hand_shape.h")]
LIB = os.path.join(HERE, "libmyo_b200.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-shared",
              "-Xcompiler", "-fPIC"]


# Verification builds of the same source (loaded by abi.lib(variant)); "f64rows": contact Jacobian rows and regularisers stored in f64
# instead of f32 -- the parity tests run both, so that storage rounding and algorithmic agreement are measured separately.
VARIANTS = {"f64rows": ["MYO_F64_ROWS"]}


def variant_path(tag):
    return os.path.join(HERE, "libmyo_b200_%s.so" % tag)


def needs_build(lib=None):
    lib = lib or LIB
    return (not os.path.exists(lib)) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in DEPS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB, SRC]
    subprocess.check_call(cmd)
    return LIB


def build_variant(tag, defines, verbose=False):
    """libmyo_b200_<tag>.so with extra -D flags (VARIANTS above)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    out = variant_path(tag)
    subprocess.check_call([nvcc] + NVCC_FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-o", out, SRC])
    return out


def build_all(force=False):
    """Product library and every verification variant, compiled concurrently (one nvcc process each, ~2 min wall-clock)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    jobs = []
    if force or needs_build():
        jobs.append((LIB, subprocess.Popen([nvcc] + NVCC_FLAGS + ["-o", LIB, SRC])))
    for tag, defs in VARIANTS.items():
        if force or needs_build(variant_path(tag)):
            jobs.append((variant_path(tag), subprocess.Popen([nvcc] + NVCC_FLAGS + ["-D" + d for d in defs] + ["-o", variant_path(tag), SRC])))
    for out, pr in jobs:
        if pr.wait() != 0:
            raise subprocess.CalledProcessError(pr.returncode, "nvcc -> " + out)
    return [LIB] + [variant_path(tag) for tag in VARIANTS]


if __name__ == "__main__":
    print(build(force=True, verbose=True))
