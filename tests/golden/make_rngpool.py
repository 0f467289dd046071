#!/usr/bin/env python
"""Generate ``reference_rngpool.npz``: the random stream of the reference's OWN ``RNGPool`` (``src/utils/utils.py:28-49``,
the class body extracted with ``ast`` and executed against numpy and ``collections.deque``), driven the way its Langevin
run drives it (``simulator.py:107-137``: ``RNGPool(seed, (n, 3), count=2)``, each step drains xi then eta and the
observer refills the pool).  Runs ONLY in the authoring container (needs /root/reference).

    python tests/golden/make_rngpool.py

For n = the protein atom counts of Chignolin and Trp-cage and seeds 0 and 2**31 - 1:

* ``state_<n>_<seed>``  uint64 [1001, 2]: (hi, lo) of the pool generator's PCG64 state after construction (row 0) and
                        after each of 1,000 drain-2 / fill-2 steps.  The pool runs two arrays ahead of the step, so row c
                        is the state after the normals of c + 1 steps.
* ``inc_<n>_<seed>``    uint64 [2]: the increment.
* ``normals_<n>_<seed>`` float64 [4, 2, n, 3]: the xi, eta the first 4 steps drained.
* ``numpy_version``     the numpy that made them: generator streams are not promised stable across releases.
"""
import ast
import collections
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))
REF = "/root/reference"

from ai2bmd_b200.fixtures import load_protein   # noqa: E402

SEEDS = (0, 2**31 - 1)
STEPS = 1000


def reference_rngpool():
    tree = ast.parse(open(f"{REF}/src/utils/utils.py").read())
    node = [n for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and n.name == "RNGPool"][0]
    ns = {"np": np, "deque": collections.deque}
    exec(compile(ast.Module(body=[node], type_ignores=[]), "ref_utils", "exec"), ns)
    return ns["RNGPool"]


def main():
    RNGPool = reference_rngpool()
    out = {"numpy_version": np.array(np.__version__)}
    for name in ("chig", "trpcage"):
        n = len(load_protein(name)[0])
        for seed in SEEDS:
            pool = RNGPool(seed=seed, shape=(n, 3), count=2)
            st = lambda: int(pool.rng.bit_generator.state["state"]["state"])     # noqa: E731
            states, normals = [st()], []
            for step in range(STEPS):
                xi = pool.standard_normal((n, 3))
                eta = pool.standard_normal((n, 3))
                if step < 4:
                    normals.append(np.stack([xi, eta]))
                pool.fill()                   # MDObserver.fill_rng_pool, attached with interval=1
                states.append(st())
            key = f"{n}_{seed}"
            out[f"state_{key}"] = np.array([[s >> 64, s & (2**64 - 1)] for s in states], dtype=np.uint64)
            inc = int(pool.rng.bit_generator.state["state"]["inc"])
            out[f"inc_{key}"] = np.array([inc >> 64, inc & (2**64 - 1)], dtype=np.uint64)
            out[f"normals_{key}"] = np.stack(normals)
    np.savez_compressed(os.path.join(HERE, "reference_rngpool.npz"), **out)


if __name__ == "__main__":
    main()
