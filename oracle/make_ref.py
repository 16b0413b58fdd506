"""Stage the UNMODIFIED reference (`/root/reference/src`, pure Python: no build step) under `oracle/_ref/` so that
it travels to the GPU box with the repo snapshot (`oracle/_ref/` is git-ignored, NOT gpurun-ignored: the sources never
enter this repository's history).

TEST / BENCH INFRASTRUCTURE.  `/root/reference` does not exist on the GPU box; `bench.py --impl reference` and the
`gpu_reference` leg import `oracle/_ref/src/*` there (through `oracle/ref_shims.py`, which only patches the library
symbols that transformers 5.x / the missing faiss removed - the reference files themselves are byte-identical copies;
`MANIFEST.json` records their sha256).  The reference has no setup.py, so the base contract's
`pip install ... /root/reference` does not apply; this copy is the tier's `oracle/_ref` equivalent.

Run in the build container:  python oracle/make_ref.py      (also called by __graft_entry__.build()).
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
DST = os.path.join(HERE, "_ref")


def stage(reference_root=REF, dst=DST, quiet=False):
    src = os.path.join(reference_root, "src")
    if not os.path.isdir(src):
        if not quiet:
            print(f"make_ref: {src} not present (GPU box?): keeping whatever is staged under {dst}")
        return os.path.isdir(os.path.join(dst, "src"))
    if os.path.isdir(dst):
        shutil.rmtree(dst)
    os.makedirs(dst)
    shutil.copytree(src, os.path.join(dst, "src"), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    manifest = {}
    for root, _, files in os.walk(os.path.join(dst, "src")):
        for f in sorted(files):
            p = os.path.join(root, f)
            with open(p, "rb") as fh:
                manifest[os.path.relpath(p, dst)] = hashlib.sha256(fh.read()).hexdigest()
    with open(os.path.join(dst, "MANIFEST.json"), "w") as fh:
        json.dump({"source": src, "files": manifest}, fh, indent=1, sort_keys=True)
    if not quiet:
        print(f"make_ref: staged {len(manifest)} reference files under {dst}")
    return True


def available(dst=DST):
    return os.path.isfile(os.path.join(dst, "src", "index.py"))


if __name__ == "__main__":
    ok = stage()
    sys.exit(0 if ok else 1)
