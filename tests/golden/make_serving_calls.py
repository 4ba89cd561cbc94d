"""Writes tests/golden/serving_calls.json: the engine calls, timing keys and result hashes of every case of
tests/test_serving_calls_host.py, recorded on the CPU.  Run from the repository root:

    python tests/golden/make_serving_calls.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.test_serving_calls_host import GOLDEN, record_all  # noqa: E402


def main():
    rec = record_all()
    with open(GOLDEN, "w") as f:
        json.dump(rec, f, sort_keys=True, separators=(",", ":"))
        f.write("\n")
    print(f"{GOLDEN}: {len(rec)} cases, {sum(len(r['calls']) for r in rec.values())} calls")


if __name__ == "__main__":
    main()
