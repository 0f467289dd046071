#!/usr/bin/env python
"""Generate ``reference_visnet_mode.npz`` and ``reference_visnet_mode_large.npz``: the reference's un-fragmented mode
(``--mode visnet``).  Runs ONLY in the authoring container (needs the reference tree, like ``make_golden.py``, whose
loader and evaluation it reuses).

    python tests/golden/make_visnet_mode.py

In ``--mode visnet`` the reference feeds the whole input to ViSNet as ONE graph (``ViSNetCalculator.calculate``,
``src/Calculators/visnet_calculator.py:138-155``).  The cases, each one graph in file order:

* ``chig``    -- whole Chignolin (175 atoms)
* ``trpcage`` -- whole Trp-cage (281 atoms)
* ``c1``      -- a three-residue ACE-X-NME input (BASELINE config C1), which the reference refuses to fragment
                 (``basefrag.py:76-84``) and sends to ``--mode visnet``: the second dipeptide of Trp-cage with its cap
                 groups renamed to ACE (CH3, HH31-33, C, O) and NME (N, H, CH3, HH31-33), so that it reads as a capped
                 residue; the protein fields ``c1_names`` / ``c1_resnames`` / ``c1_resnums`` / ``c1_elements`` rebuild it.

and, in ``reference_visnet_mode_large.npz`` (a file of its own, so that the first one stays as it was), the two larger
example proteins, whose one-graph plans the cases above never select (ABD crosses the 600-atom rule of the tensor-core
node stage; both run several edge tiles per CTA):

* ``ww``      -- whole WW domain (571 atoms)
* ``abd``     -- whole ABD (746 atoms)

Per case: ``<key>_z``, ``_pos`` (fp32), ``_batch`` (zeros), ``_slots`` / ``_deg`` (the canonical neighbour slots of
``oracle/radius_graph.c``, which the reference's ``radius_graph`` stand-in returns), ``_ref_e`` / ``_ref_f`` (the
reference's own model source, fp32 CPU, through ``oracle/ref_shims.py``) and ``_e64`` / ``_f64`` (the fp64 oracle).
In whole proteins most interior atoms have more than 32 atoms within 5 A, so the first-32-by-index cap truncates
routinely; the script prints the largest candidate count and the number of truncated atoms per case.  Both files are
byte-identical on every run (the evaluations are deterministic and numpy writes its zip entries without timestamps).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import CKPT, REF, load_reference_model, ref_eval          # noqa: E402
from oracle import visnet_ref as O                                         # noqa: E402
from ai2bmd_b200.pdbfrag import CappedProtein, fragment_protein, read_pdb, whole_input   # noqa: E402

# cap groups of a dipeptide renamed as the ACE / NME residues of a capped input (by the atom's name in its residue)
_ACE = {"CA": "CH3", "HA": "HH31", "C": "C", "O": "O"}
_NME = {"N": "N", "H": "H", "CA": "CH3", "HA": "HH31"}


def c1_input(prot, g=2):
    """Fragment g of ``prot`` (a dipeptide: leading cap group, centre residue, trailing cap group) as a three-residue
    ACE-X-NME CappedProtein in the fragment's atom order."""
    fd, pm, rc = fragment_protein(prot, with_recipe=True)
    a0, a1 = int(fd.start[g]), int(fd.end[g])
    res_of = lambda a: int(prot.resnums[rc.real[a] if rc.real[a] >= 0 else rc.acc[a]])     # noqa: E731
    lead, centre = res_of(a0), res_of(a0) + 1
    names, resn, resi, elem = [], [], [], []
    extra = {1: 2, 3: 2}                       # next HH3x index per cap residue
    for a in range(a0, a1):
        r = res_of(a)
        if r == centre:
            i = int(rc.real[a])
            names.append(prot.names[i]); resn.append(prot.resnames[i]); resi.append(2); elem.append(prot.elements[i])
            continue
        cap = 1 if r == lead else 3
        table = _ACE if cap == 1 else _NME
        if rc.real[a] >= 0:
            nm = table[prot.names[int(rc.real[a])]]
            el = prot.elements[int(rc.real[a])]
        else:                                  # an added hydrogen on the cap carbon
            nm, el = f"HH3{extra[cap]}", "H"
            extra[cap] += 1
        names.append(nm); resn.append("ACE" if cap == 1 else "NME"); resi.append(cap); elem.append(el)
    pos = np.asarray(fd.pos[a0:a1], dtype=np.float64)
    return CappedProtein(names, resn, np.asarray(resi, dtype=np.int64), elem, pos)


def one_graph_cases(model, o64, prots):
    """Every field of each case, the whole input as one graph."""
    out = {}
    for key, prot in prots.items():
        fd = whole_input(prot)
        assert len(fd) == 1
        e, f = ref_eval(model, fd)
        e64, f64 = o64.energy_and_forces(fd.z, fd.pos, fd.batch)
        slots, deg = O.radius_graph_canonical(fd.pos, fd.batch)
        p = np.asarray(fd.pos, dtype=np.float32)
        cand = ((p[:, None, :] - p[None, :, :]) ** 2).sum(-1) < np.float32(5.0) ** 2
        n_cand = cand.sum(1)
        out[f"{key}_z"], out[f"{key}_pos"], out[f"{key}_batch"] = fd.z, fd.pos, fd.batch
        out[f"{key}_ref_e"], out[f"{key}_ref_f"] = e, f
        out[f"{key}_e64"], out[f"{key}_f64"] = e64.numpy(), f64.numpy()
        out[f"{key}_slots"], out[f"{key}_deg"] = slots, deg
        print(f"{key}: N={len(fd.z)} E={int(deg.sum())} max candidates within 5 A={int(n_cand.max())} "
              f"truncated atoms={int((n_cand > 32).sum())} maxdeg={int(deg.max())} "
              f"|ref-o64| E {np.abs(e - e64.numpy()).max():.3e} F {np.abs(f - f64.numpy()).max():.3e}")
    return out


def main():
    sd = O.load_state_dict(CKPT)
    model = load_reference_model()
    o64 = O.OracleViSNet(sd, torch.float64)
    prots = {"chig": read_pdb(f"{REF}/examples/chig.pdb"), "trpcage": read_pdb(f"{REF}/examples/trpcage.pdb")}
    prots["c1"] = c1_input(prots["trpcage"])
    try:
        fragment_protein(prots["c1"])
        raise AssertionError("the three-residue input was fragmented")
    except NotImplementedError:
        pass
    out = one_graph_cases(model, o64, prots)
    c1 = prots["c1"]
    out.update(c1_names=np.array(c1.names), c1_resnames=np.array(c1.resnames), c1_resnums=c1.resnums,
               c1_elements=np.array(c1.elements))
    np.savez_compressed(os.path.join(HERE, "reference_visnet_mode.npz"), **out)
    # at these sizes torch's CPU backward splits its scatter-adds over threads, and the reference's fp32 forces then move
    # by an ulp or two from run to run; one thread keeps the file reproducible
    torch.set_num_threads(1)
    large = one_graph_cases(model, o64, {k: read_pdb(f"{REF}/examples/{k}.pdb") for k in ("ww", "abd")})
    np.savez_compressed(os.path.join(HERE, "reference_visnet_mode_large.npz"), **large)


if __name__ == "__main__":
    main()
