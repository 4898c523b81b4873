#!/usr/bin/env python3
"""Regenerate data/*.yaml (model INPUTS) from the reference's data directory.

The model inputs are data, not code: the basis description (number of spins, Hamming weight, spin
inversion, symmetry generators) and the Hamiltonian term list (expression + site tuples) of each
reference's data/*.yaml (kept verbatim in tests/golden/reference_data.tar.xz).  This script extracts that semantic
content and re-emits it in a normalised layout (no anchors, no comments, no solver-only keys such as `observables`,
`number_vectors`, `output`, `max_primme_*`).  tests/test_host.py (test_model_inputs_equal_the_reference_inputs)
re-checks semantic equality against the stored copies.

Usage:  python tools/gen_models.py REFERENCE_DATA_DIR [data]
        python tools/gen_models.py --fermions [data]

--fermions writes the fermionic models, which the reference's data directory does not have: hubbard_chain_8 (periodic
chain of 8 sites) and hubbard_square_4x4 (4 x 4 torus), H = -t sum_<ij>,s (c+_is c_js + h.c.) + U sum_i n_i,up n_i,down
with t = 1, U = 4 at half filling; and spinless_ring_28, H = -t sum_i (c+_i c_i+1 + h.c.) with t = 1 at 14 particles.
Each also in one symmetry sector (site_symmetries): spinless_ring_28_symm (translations, momentum 0),
hubbard_chain_8_symm (translations and the reflection i -> 7 - i, both sector 0) and hubbard_square_4x4_symm (the two
torus translations, momentum (0, 0)).
"""
import glob
import os
import sys

import yaml


class _Flow(list):
    pass


def _flow_representer(dumper, data):
    return dumper.represent_sequence("tag:yaml.org,2002:seq", data, flow_style=True)


yaml.add_representer(_Flow, _flow_representer, Dumper=yaml.SafeDumper)


def normalise(conf: dict) -> dict:
    b = conf["basis"]
    basis = {
        "number_spins": int(b["number_spins"]),
        "hamming_weight": b.get("hamming_weight", None),
        "spin_inversion": b.get("spin_inversion", None),
        "symmetries": [
            {"permutation": _Flow(int(v) for v in g["permutation"]), "sector": int(g.get("sector", 0))}
            for g in (b.get("symmetries") or [])
        ],
    }
    terms = []
    for t in conf["hamiltonian"]["terms"]:
        entry = {}
        if "expression" in t:
            entry["expression"] = t["expression"]
        else:
            entry["matrix"] = [_Flow(row) for row in t["matrix"]]
        entry["sites"] = _Flow(_Flow(int(s) for s in tup) for tup in t["sites"])
        terms.append(entry)
    return {"basis": basis, "hamiltonian": {"name": conf["hamiltonian"].get("name", ""), "terms": terms}}


def _bonds_ring(n):
    return [[i, (i + 1) % n] for i in range(n)]


def _bonds_torus(lx, ly):
    out = []
    for y in range(ly):
        for x in range(lx):
            i = x + lx * y
            out += [[i, (x + 1) % lx + lx * y], [i, x + lx * ((y + 1) % ly)]]
    return out


def hubbard(n_sites, bonds, t=1.0, u=4.0, number_up=None, number_down=None, name="Hubbard model"):
    up = n_sites // 2 if number_up is None else number_up
    down = n_sites // 2 if number_down is None else number_down
    hop = f"-{t} × c†₀↑ c₁↑ - {t} × c†₁↑ c₀↑ - {t} × c†₀↓ c₁↓ - {t} × c†₁↓ c₀↓"
    return {"basis": {"particle": "spinful-fermion", "number_sites": n_sites, "number_particles": up + down,
                      "number_up": up},
            "hamiltonian": {"name": name, "terms": [
                {"expression": hop, "sites": _Flow(_Flow(b) for b in bonds)},
                {"expression": f"{u} × n₀↑ n₀↓", "sites": _Flow(_Flow([i]) for i in range(n_sites))}]}}


def spinless_ring(n_sites, number_particles, t=1.0, name="spinless fermions on a ring"):
    return {"basis": {"particle": "spinless-fermion", "number_sites": n_sites, "number_particles": number_particles},
            "hamiltonian": {"name": name, "terms": [
                {"expression": f"-{t} × c†₀ c₁ - {t} × c†₁ c₀", "sites": _Flow(_Flow(b) for b in _bonds_ring(n_sites))}]}}


def ring_translation(n):
    return [(i + 1) % n for i in range(n)]


def ring_reflection(n):
    return [n - 1 - i for i in range(n)]


def torus_translations(lx, ly):
    """x -> x + 1 and y -> y + 1 on the sites i = x + lx y of _bonds_torus"""
    return ([(x + 1) % lx + lx * y for y in range(ly) for x in range(lx)],
            [x + lx * ((y + 1) % ly) for y in range(ly) for x in range(lx)])


def with_site_symmetries(conf, permutations, sectors=None):
    """conf with basis.site_symmetries = the permutations, in the given sectors (default 0)"""
    sectors = [0] * len(permutations) if sectors is None else sectors
    out = {"basis": dict(conf["basis"]), "hamiltonian": conf["hamiltonian"]}
    out["basis"]["site_symmetries"] = [{"permutation": _Flow(p), "sector": int(k)} for p, k in zip(permutations, sectors)]
    return out


def fermion_models() -> dict:
    return {"hubbard_chain_8": hubbard(8, _bonds_ring(8)),
            "hubbard_square_4x4": hubbard(16, _bonds_torus(4, 4)),
            "spinless_ring_28": spinless_ring(28, 14),
            "spinless_ring_28_symm": with_site_symmetries(spinless_ring(28, 14), [ring_translation(28)]),
            "hubbard_chain_8_symm": with_site_symmetries(hubbard(8, _bonds_ring(8)),
                                                         [ring_translation(8), ring_reflection(8)]),
            "hubbard_square_4x4_symm": with_site_symmetries(hubbard(16, _bonds_torus(4, 4)),
                                                            list(torus_translations(4, 4)))}


def write_fermion_models(dst):
    for name, conf in fermion_models().items():
        with open(os.path.join(dst, name + ".yaml"), "w", encoding="utf-8") as f:
            f.write(f"# model input '{name}.yaml': written by tools/gen_models.py --fermions\n")
            yaml.safe_dump(conf, f, allow_unicode=True, sort_keys=False, width=120)
        print("wrote", name)


def main():
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    if sys.argv[1] == "--fermions":
        write_fermion_models(sys.argv[2] if len(sys.argv) > 2 else os.path.join(os.path.dirname(__file__), "..", "data"))
        return
    src = sys.argv[1]
    dst = sys.argv[2] if len(sys.argv) > 2 else os.path.join(os.path.dirname(__file__), "..", "data")
    os.makedirs(dst, exist_ok=True)
    for path in sorted(glob.glob(os.path.join(src, "*.yaml"))):
        with open(path, "r", encoding="utf-8") as f:
            conf = yaml.safe_load(f)
        out = normalise(conf)
        name = os.path.basename(path)
        with open(os.path.join(dst, name), "w", encoding="utf-8") as f:
            f.write(f"# model input '{name}': normalised by tools/gen_models.py (see its docstring)\n")
            yaml.safe_dump(out, f, allow_unicode=True, sort_keys=False, width=120)
        print("wrote", name)


if __name__ == "__main__":
    main()
