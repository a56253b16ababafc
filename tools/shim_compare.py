"""Run the drop-in boundary checks of tests/test_gpu_shim.py outside pytest and print each build's timings.

    python tools/shim_compare.py

The checks themselves live in the test module (one copy); this only runs them one by one on a GPU, after oracle/ref_shim.mk has built
oracle/_ref/shim, and prints the reference build's and the shim build's *_ms / *_gcups figures side by side."""
import os
import sys
import tempfile

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests import test_gpu_shim as T  # noqa: E402


def main():
    failed = 0
    for check in T.CHECKS:
        with tempfile.TemporaryDirectory() as tmp:
            try:
                ref, b2 = check(tmp)
            except AssertionError as e:
                failed += 1
                print("FAIL", check.__name__, e)
                continue
            except pytest.skip.Exception as e:         # a binary is not built
                failed += 1
                print("SKIP", check.__name__, e)
                continue
            timing = lambda r: {k: v for k, v in r.items() if k.endswith("_ms") or k.endswith("gcups")}
            print("ok  ", check.__name__, "reference", timing(ref), "shim", timing(b2))
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
