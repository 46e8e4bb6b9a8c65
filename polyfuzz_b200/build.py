"""Build libpfz.so (all CUDA kernels + the C ABI) for sm_90a with nvcc, in-tree.

    python -m polyfuzz_b200.build [--force]

The shared library is self-contained (static cudart), exports only the extern "C" symbols declared
in include/pfz.h, and is what every GPU code path of this package calls through ctypes.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libpfz.so")
SOURCES = ["pfz_core.cu", "pfz_tfidf.cu", "pfz_spcos.cu", "pfz_spcos_block.cu", "pfz_spcos_hash.cu", "pfz_lev.cu", "pfz_fuzz.cu", "pfz_tok.cu", "pfz_dense.cu", "pfz_assemble.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    deps.append(os.path.join(HERE, "..", "include", "pfz.h"))
    return any(os.path.getmtime(d) > t for d in deps)


HOSTPACK_SRC = os.path.join(CSRC, "pfz_hostpack.c")


def hostpack_path():
    import sysconfig
    return os.path.join(HERE, "_pfz_hostpack" + (sysconfig.get_config_var("EXT_SUFFIX") or ".so"))


def build_hostpack(force=False):
    """The small CPython extension that packs list[str] into blob + offsets (host marshalling, plain gcc)."""
    import sysconfig
    out = hostpack_path()
    if not force and os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(HOSTPACK_SRC):
        return out
    env = dict(os.environ); env.pop("CC", None)
    cmd = ["gcc", "-O3", "-fPIC", "-shared", "-I", sysconfig.get_paths()["include"], "-o", out, HOSTPACK_SRC]
    res = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if res.returncode != 0:
        raise RuntimeError("gcc failed for pfz_hostpack.c:\n" + res.stdout + res.stderr)
    return out


def build(force=False, verbose=False):
    build_hostpack(force)
    if not force and not needs_build():
        return LIB
    import concurrent.futures
    import tempfile
    extra = os.environ.get("PFZ_NVCC_EXTRA", "").split()          # developer builds (e.g. -DPFZ_B3_TIMING)
    env = dict(os.environ)
    # the image's CC wrapper lacks OpenMP specs; nvcc only needs a plain host g++
    env.pop("CC", None); env.pop("CXX", None)
    with tempfile.TemporaryDirectory(prefix="pfz_build_") as tmp:
        # the translation units share no device code: compile them in parallel, then link once
        objs = [os.path.join(tmp, os.path.basename(s)[:-3] + ".o") for s in sources()]
        cmds = [[_nvcc()] + NVCC_FLAGS + extra + ["-c", "-o", o, s] for s, o in zip(sources(), objs)]
        tmp_lib = os.path.join(tmp, "libpfz.so")
        link = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "--shared", "-o", tmp_lib] + objs
        with concurrent.futures.ThreadPoolExecutor(max_workers=min(len(cmds), os.cpu_count() or 1)) as ex:
            results = list(ex.map(lambda c: subprocess.run(c, capture_output=True, text=True, env=env), cmds))
        log = "".join(" ".join(c) + "\n" + r.stdout + r.stderr for c, r in zip(cmds, results))
        failed = any(r.returncode != 0 for r in results)
        if not failed:
            r = subprocess.run(link, capture_output=True, text=True, env=env)
            log += " ".join(link) + "\n" + r.stdout + r.stderr
            failed = r.returncode != 0
        with open(os.path.join(HERE, "build.log"), "w") as f:
            f.write(log)
        if failed:
            raise RuntimeError("nvcc failed:\n" + log[-4000:])
        _copy(tmp_lib, LIB)
    if verbose:
        print(log)
    return LIB


def _copy(src, dst):
    """Copy next to dst, then rename: a reader never sees a half-written library."""
    import shutil
    part = dst + ".part"
    shutil.copyfile(src, part)
    os.chmod(part, 0o755)
    os.replace(part, dst)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
