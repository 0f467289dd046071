#!/usr/bin/env python
"""Generate ``reference_chunks.json``.  Runs ONLY in the authoring container (needs /root/reference).

    python tests/golden/make_reference_chunks.py

Writes, next to this file, ``reference_chunks.json``: (device, first fragment, end fragment) of every chunk the
reference's OWN work-partition function (``DeviceStrategy._set_combined_work_partitions``,
``src/Calculators/device_strategy.py:83-125``, extracted with ``ast`` because the module imports ase) cuts with
``_chunk_size`` 40 / 100 / 250 / 1000 atoms at 1/2/4 devices, for the four example proteins (fragments as committed in
``fragments_<prot>.npz``).  Every chunk size is at least the largest fragment (36 atoms), so the reference's loop ends.
The other goldens are written by ``make_golden.py``; this script reads and rewrites none of them.
"""
import ast
import bisect
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
REF = "/root/reference"

from ai2bmd_b200.fixtures import load_fragments   # noqa: E402


def reference_work_partitions():
    """The reference's ``_set_combined_work_partitions(cls, devices, start, end)``: stores ``[(device, first, end)]`` in
    ``cls._work_partitions``, blocks per device cut into chunks of ``cls._chunk_size`` atoms."""
    tree = ast.parse(open(f"{REF}/src/Calculators/device_strategy.py").read())
    fn = [n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "_set_combined_work_partitions"][0]
    fn.decorator_list = []
    ns = {"bisect": bisect}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "ref_device_strategy", "exec"), ns)
    return ns["_set_combined_work_partitions"]


def main():
    fn = reference_work_partitions()

    class Cls:
        _chunk_size = None
        _work_partitions = None

    out = {}
    for name in ("chig", "trpcage", "ww", "abd"):
        fd, _ = load_fragments(name)
        start, end = [int(x) for x in fd.start], [int(x) for x in fd.end]
        assert 40 >= max(e - s for s, e in zip(start, end))       # else the reference's chunk loop never ends
        for n in (1, 2, 4):
            for chunk in (40, 100, 250, 1000):
                Cls._chunk_size = chunk
                fn(Cls, list(range(n)), start, end)
                out[f"{name}:{n}:{chunk}"] = [[int(d), int(a), int(b)] for d, a, b in Cls._work_partitions]
    with open(os.path.join(HERE, "reference_chunks.json"), "w") as fh:
        json.dump(out, fh, sort_keys=True)


if __name__ == "__main__":
    main()
