#!/usr/bin/env python
"""Install the UNMODIFIED reference project next to the oracle: reference checkout -> oracle/_ref/.

`oracle/_ref/` is git-ignored: the reference's sources never enter this repository.  The reference has no setup.py /
pyproject.toml, so there is nothing to pip-install; this recipe copies its Python sources and `hyperparam.ini`
verbatim (no edits -- `tests/test_reference_shipping.py` checks the copies byte for byte against the SHA-256 digests
of the reference's files stored in tests/golden/reference_digests.json).  `__graft_entry__.build()` runs it; the
checkout is read from $DISVAE_REFERENCE (default: the build host's reference checkout, DEFAULT_REF); where neither
exists it keeps whatever oracle/_ref holds.

Used by: `bench.py --impl reference` / `--impl reference-cuda` (the reference's own Trainer on the host cores / on
the GPU through stock PyTorch eager) and `tests/test_main_gpu.py` (the reference's `main.py` driving this
repository's `disvae` package).

    python oracle/ship_reference.py                   # copy the reference into oracle/_ref
    python oracle/ship_reference.py --digests OUT     # write the digest table of the reference checkout to OUT
"""
import hashlib
import json
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_REF = "/root/reference"
REF = os.environ.get("DISVAE_REFERENCE", DEFAULT_REF)
DST = os.path.join(ROOT, "oracle", "_ref")
ITEMS = ["disvae", "utils", "main.py", "main_viz.py", "hyperparam.ini", "LICENSE"]


def digest_table(root):
    """{relative path: sha256} of the reference's Python sources under disvae/ and utils/ and of its top-level
    main.py, main_viz.py and hyperparam.ini (the files this repository's tests and bench arms run)."""
    files = []
    for base in ("disvae", "utils"):
        for d, _, names in os.walk(os.path.join(root, base)):
            files += [os.path.join(d, f) for f in names if f.endswith(".py")]
    files += [os.path.join(root, f) for f in ("main.py", "main_viz.py", "hyperparam.ini")]
    table = {}
    for f in sorted(files):
        with open(f, "rb") as fh:
            table[os.path.relpath(f, root)] = hashlib.sha256(fh.read()).hexdigest()
    return table


def ship(verbose=True):
    if not REF or not os.path.isdir(REF):
        if verbose:
            print("no reference checkout at %s: keeping whatever oracle/_ref holds" % REF)
        return os.path.isdir(os.path.join(DST, "disvae"))
    os.makedirs(DST, exist_ok=True)
    for it in ITEMS:
        src, dst = os.path.join(REF, it), os.path.join(DST, it)
        if os.path.isdir(src):
            if os.path.isdir(dst):
                shutil.rmtree(dst)
            shutil.copytree(src, dst, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
        else:
            shutil.copyfile(src, dst)
    if verbose:
        print("reference shipped to", DST)
    return True


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--digests":
        with open(sys.argv[2], "w") as fh:
            json.dump(digest_table(REF), fh, indent=1, sort_keys=True)
            fh.write("\n")
        sys.exit(0)
    sys.exit(0 if ship() else 1)
