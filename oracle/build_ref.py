"""Build the reference binaries that the reference-side harness (`baseline/refenv.py`) runs, into oracle/_ref/:

    oracle/_ref/HairFastGAN/   the reference checkout compiled to sourceless bytecode: one `.pyc` where each `.py`
                               was, plus the checkout's data files (configs, style codes, images); no source file
    oracle/_ref/ext/<name>/    its two JIT CUDA extensions (models/stylegan2/op/fused_act.py:10-16,
                               upfirdn2d.py:10-16), built for sm_90 by torch's own extension builder

The checkout is looked up in this order: the directory named by HAIRFAST_REFERENCE; a directory `reference` beside
this repository or beside any directory above it; the reference's standard mount point, /root/reference (see
`MOUNT_POINT`).  Without one nothing is built and the harness reports the reference as unavailable.  The sources are compiled from a temporary
copy; nothing of them is written under this repository.

    python oracle/build_ref.py [--force]
"""
from __future__ import annotations

import compileall
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(HERE, "_ref")
TREE = os.path.join(OUT, "HairFastGAN")
EXT = os.path.join(OUT, "ext")
DATA_SUFFIXES = (".npy", ".yaml", ".yml", ".json", ".txt", ".webp", ".png", ".jpg")
MOUNT_POINT = "/root/reference"       # where the build image mounts the read-only reference checkout
EXTENSIONS = {"fused": ("fused_bias_act.cpp", "fused_bias_act_kernel.cu"),
              "upfirdn2d": ("upfirdn2d.cpp", "upfirdn2d_kernel.cu")}


def _candidates():
    yield os.environ.get("HAIRFAST_REFERENCE")
    d = ROOT
    while os.path.dirname(d) != d:
        d = os.path.dirname(d)
        yield os.path.join(d, "reference")
    yield MOUNT_POINT


def find_checkout() -> str | None:
    for cand in _candidates():
        try:
            if cand and os.path.isfile(os.path.join(cand, "hair_swap.py")):
                return os.path.abspath(cand)
        except OSError:            # an ancestor the building user may not list
            continue
    return None


def built() -> bool:
    return os.path.isfile(os.path.join(TREE, "hair_swap.pyc")) and all(
        os.path.isfile(os.path.join(EXT, n, n + ".so")) for n in EXTENSIONS)


def _build_extensions(src_tree: str) -> None:
    """torch.utils.cpp_extension.load of both extensions, in a child process (the builder caches per process)."""
    op = os.path.join(src_tree, "models", "stylegan2", "op")
    code = ("import sys, torch\nfrom torch.utils.cpp_extension import load\n"
            "for name, srcs in %r.items():\n"
            "    load(name, sources=[%r + '/' + s for s in srcs])\n" % (EXTENSIONS, op))
    env = dict(os.environ, TORCH_EXTENSIONS_DIR=EXT, TORCH_CUDA_ARCH_LIST=os.environ.get("TORCH_CUDA_ARCH_LIST", "9.0"))
    env.setdefault("MAX_JOBS", "8")
    subprocess.run([sys.executable, "-c", code], check=True, env=env, timeout=1800, stdout=subprocess.DEVNULL)


def build(force: bool = False) -> str | None:
    """Returns the bytecode tree, or None when no reference checkout is found."""
    if built() and not force:
        return TREE
    src = find_checkout()
    if src is None:
        return None
    with tempfile.TemporaryDirectory() as tmp:
        work = os.path.join(tmp, "HairFastGAN")
        shutil.copytree(src, work, ignore=shutil.ignore_patterns(".git", "__pycache__"), copy_function=shutil.copyfile)
        for dirpath, _, _ in os.walk(work):                       # a read-only checkout gives read-only directories
            os.chmod(dirpath, 0o755)
        compileall.compile_dir(work, quiet=2, legacy=True)       # legacy: foo.pyc beside foo.py, importable alone
        if not os.path.isfile(os.path.join(work, "hair_swap.pyc")):
            raise RuntimeError(f"compiling the reference checkout {src} to bytecode failed")
        shutil.rmtree(OUT, ignore_errors=True)
        for dirpath, _, files in os.walk(work):
            rel = os.path.relpath(dirpath, work)
            for f in files:
                if f.endswith(".pyc") or f.lower().endswith(DATA_SUFFIXES):
                    os.makedirs(os.path.join(TREE, rel), exist_ok=True)
                    shutil.copy2(os.path.join(dirpath, f), os.path.join(TREE, rel, f))
        _build_extensions(work)
    return TREE


if __name__ == "__main__":
    print(build(force="--force" in sys.argv) or "no reference checkout found")
