"""oracle/_ref must be the reference byte for byte: every file of the stored digest table of the reference
(tests/golden/reference_digests.json, SHA-256 of the reference's sources) against the copy oracle/ship_reference.py
made (CPU test; the copy exists where build() found a reference checkout)."""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")


def test_shipped_reference_is_unmodified():
    if not os.path.isdir(DST):
        pytest.skip("oracle/_ref not shipped")
    from oracle import ship_reference
    with open(os.path.join(ROOT, "tests", "golden", "reference_digests.json")) as fh:
        want = json.load(fh)
    got = ship_reference.digest_table(DST)
    assert got == want, sorted(k for k in set(got) | set(want) if got.get(k) != want.get(k))
    assert sum(k.endswith(".py") for k in want) > 15
    assert {"main.py", "main_viz.py", "hyperparam.ini"} <= set(want)


def test_reference_imports_from_shipped_copy():
    if not os.path.isdir(DST):
        pytest.skip("oracle/_ref not shipped")
    import subprocess
    import sys
    code = ("import sys; sys.path.insert(0, %r); from oracle import reference_env as E; d = E.activate(%r); "
            "import disvae, os; assert os.path.realpath(disvae.__file__).startswith(os.path.realpath(d)); "
            "from disvae.training import Trainer; import main; print('ok')" % (ROOT, DST))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]
