#!/usr/bin/env python
"""Generate ``reference_hbond_pairs.json``.  Runs ONLY in the authoring container (needs /root/reference), like
``make_golden.py`` next to it.

    python tests/golden/make_hbond_pairs.py

Hydrogen bond constraint pairs (i_H, j, rt, k) of the reference's OWN ``PDBAnalyzer.find_bonded_atoms("H")``
(``src/utils/utils.py:184-221``, what ``--constraints`` adds as springs, ``src/AIMD/simulator.py:168-180``; the class is
extracted with ``ast`` because the module imports torch / ase / AIMD.arguments, and needs numpy only) for the four example
proteins and the pre-equilibrated Chignolin, stored with the ATOM names and coordinates the class parsed, so the tests
(``tests/test_restraints.py``) need no reference tree.  Data only.
"""
import ast
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
PDBS = {"chig": "examples/chig.pdb", "trpcage": "examples/trpcage.pdb", "ww": "examples/ww.pdb",
        "abd": "examples/abd.pdb", "chig_preeq_nowat": "examples/chig_preprocessed/chig-preeq-nowat.pdb"}


def main():
    tree = ast.parse(open(f"{REF}/src/utils/utils.py").read())
    cls = [n for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and n.name == "PDBAnalyzer"][0]
    ns = {"np": np}
    exec(compile(ast.Module(body=[cls], type_ignores=[]), "ref_utils", "exec"), ns)
    out = {}
    for key, rel in PDBS.items():
        an = ns["PDBAnalyzer"](f"{REF}/{rel}")
        pairs = an.find_bonded_atoms("H")
        out[key] = {"names": [a[0] for a in an.atoms], "positions": [[float(c) for c in a[1]] for a in an.atoms],
                    "pairs": [[int(i), int(j), float(rt), float(k)] for i, j, rt, k in pairs]}
        print(f"hydrogen bond pairs ({key}): {len(pairs)} for {len(an.atoms)} atoms")
    with open(os.path.join(HERE, "reference_hbond_pairs.json"), "w") as fh:
        json.dump(out, fh, sort_keys=True)


if __name__ == "__main__":
    main()
