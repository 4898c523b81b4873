#!/usr/bin/env python3
"""How often does an off-diagonal target of a row share its leading key bits with the row's own representative?
That is the locality the ordered table layout of k_rows (rows_table = 1) turns into L2 hits: the rows run in ascending
key order, and the table is laid out by key prefix.  CPU only: representatives and targets are canonicalised by the
library's host-side self-check entry (the device functions compiled for the host).

Samples random S_z = 0 states, canonicalises them (the sampled rows), canonicalises every off-diagonal target of each,
and prints per prefix length the fraction of targets that share the row's prefix and the largest prefix block (share of
the sampled representatives).  Prefixes count from the highest bit any sampled representative uses.  With
--bytes-per-state B it also prints a model estimate of the L2 hit fraction: a target hits when its rank in the sorted
basis lies within the window of L2 / B states around the row's rank (ranks estimated from the sample).

Usage: python tools/lookup_locality.py MODEL [SAMPLE] [--bytes-per-state B] [--l2-mb 50] [--bits 14]"""
import argparse
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from distributed_matvec_b200 import _native as nat  # noqa: E402
from distributed_matvec_b200.config import load_config_from_yaml  # noqa: E402


def canonicalise(basis, states):
    g = basis.group
    bd = nat.BasisDesc()
    bd.number_sites, bd.hamming_weight, bd.spin_inversion, bd.has_permutations = (
        basis.number_sites, -1 if basis.hamming_weight is None else basis.hamming_weight, basis.spin_inversion, 1)
    perms, flips, chars = (np.ascontiguousarray(g.perms), np.ascontiguousarray(g.flips),
                           np.ascontiguousarray(g.characters))
    bd.group_order, bd.perms, bd.flips, bd.characters = len(g), perms.ctypes.data, flips.ctypes.data, chars.ctypes.data
    states = np.ascontiguousarray(states, dtype=np.uint64)
    reps = np.zeros_like(states)
    nat.check(nat.lib().dmv_debug_compile_group(C.byref(bd), None, states.shape[0], states.ctypes.data,
                                                reps.ctypes.data, None))
    return reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("model")
    ap.add_argument("sample", type=int, nargs="?", default=20000)
    ap.add_argument("--bytes-per-state", type=float, default=0.0)
    ap.add_argument("--l2-mb", type=float, default=50.0)
    ap.add_argument("--states", type=float, default=0.0, help="basis size (needed for the L2 estimate)")
    ap.add_argument("--bits", type=int, default=14, help="directory bits for the block-size distribution")
    args = ap.parse_args()
    basis, matrix = load_config_from_yaml(os.path.join(ROOT, "data", args.model + ".yaml"))
    n = basis.number_sites
    rng = np.random.default_rng(1)
    w = basis.hamming_weight if basis.hamming_weight is not None else n // 2
    states = np.zeros(args.sample, dtype=np.uint64)
    for k in range(args.sample):
        for site in rng.choice(n, size=w, replace=False):
            states[k] |= np.uint64(1) << np.uint64(site)
    rows = canonicalise(basis, states)
    off = matrix.off_diag
    m, r, x = (np.asarray(off.m, dtype=np.uint64), np.asarray(off.r, dtype=np.uint64),
               np.asarray(off.x, dtype=np.uint64))
    emit = (rows[:, None] & m[None, :]) == r[None, :]
    row_of, term = np.nonzero(emit)
    targets = canonicalise(basis, rows[row_of] ^ x[term])
    top = int(max(int(rows.max()), int(targets.max()))).bit_length()
    print(f"{args.model}: {args.sample} sampled rows, {targets.shape[0]} off-diagonal targets "
          f"({targets.shape[0] / args.sample:.1f} per row), keys use {top} bits")
    print("shared prefix  targets sharing it  largest block (share of rows)")
    for p in (8, 10, 12, 14, 16, 18):
        s = np.uint64(max(0, top - p))
        same = float(np.mean((targets >> s) == (rows[row_of] >> s)))
        _, counts = np.unique(rows >> s, return_counts=True)
        print(f"  {p:2d} bits        {100 * same:6.1f} %            {100 * counts.max() / args.sample:6.2f} %")
    # block sizes of the directory the ordered layout would use (ordered_plan: 2^bits blocks over [k_lo, k_hi])
    srt = np.sort(rows)
    span = int(srt[-1] - srt[0])
    shift = max(0, span.bit_length() - args.bits)
    _, counts = np.unique((srt - srt[0]) >> np.uint64(shift), return_counts=True)
    share = counts / args.sample
    print(f"directory of 2^{args.bits} blocks (shift {shift}): {counts.shape[0]} non-empty blocks in the sample; "
          f"share of states per block: median {np.median(share):.2e}, 99 % {np.quantile(share, 0.99):.2e}, "
          f"max {share.max():.2e}")
    if args.bytes_per_state > 0 and args.states > 0:
        window = args.l2_mb * 2**20 / args.bytes_per_state / args.states   # L2 window as a fraction of the basis
        rank_row = np.searchsorted(srt, rows[row_of]) / args.sample
        rank_t = np.searchsorted(srt, targets) / args.sample
        hit = float(np.mean(np.abs(rank_t - rank_row) < window / 2))
        print(f"L2 window {args.l2_mb:.0f} MB at {args.bytes_per_state:.0f} B per state = {100 * window:.2f} % of "
              f"{args.states:.0f} states: estimated hit fraction {100 * hit:.1f} % (model, not measured)")


if __name__ == "__main__":
    main()
