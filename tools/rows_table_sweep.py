#!/usr/bin/env python3
"""Time k_rows with the hashed and the ordered layout of its look-up table (rows_table = 0 / 1), the ordered one at
several directory sizes (rows_table_bits) and, for complex128, buckets per state (rows_table_buckets), each ordered
configuration with every asked L2 eviction mode (rows_l2) and window (rows_l2_window, MB; modes other than 0), and the
dense ordered table (rows_dense_order = 1: one slot per state in key order) at every asked directory size (--dense-bits)
with every asked L2 mode and window (--dense-windows); every configuration at every asked number of CTAs per SM of
k_rows (--ctas: rows_ctas, -1 auto), with the CTAs the launch had resident.  The configurations alternate in rounds; each
product is timed with CUDA events, the L2 flushed before it, and every configuration's y is compared with the first's
(the hashed layout's unless --no-hashed) by the element criterion of bench.py.
Usage: python tools/rows_table_sweep.py [--rounds R] [--products K] [workload ...]"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributed_matvec_b200 import Operator, load_config_from_yaml  # noqa: E402

def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError as e:
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--products", type=int, default=6, help="timed products per configuration and round")
    ap.add_argument("--dtypes", default="c128,f64")
    ap.add_argument("--bits", default="10,12,14", help="directory sizes of the ordered layout (rows_table_bits; empty: not timed)")
    ap.add_argument("--buckets", default="2,4,8", help="complex128 buckets per state of the ordered layout")
    ap.add_argument("--l2", default="0", help="L2 eviction modes of the ordered layout (rows_l2)")
    ap.add_argument("--l2-window", default="16", help="near windows in MB of table (rows_l2_window)")
    ap.add_argument("--dense-windows", default="", help="near windows in MB of the dense ordered table (empty: not timed)")
    ap.add_argument("--dense-bits", default="14", help="directory sizes of the dense ordered table (rows_table_bits)")
    ap.add_argument("--no-hashed", action="store_true",
                    help="leave the hashed layout out: the first configuration is then the reference of times and y")
    ap.add_argument("--ctas", default="2", help="CTAs per SM of k_rows (rows_ctas; -1: auto)")
    ap.add_argument("workloads", nargs="*", default=["heisenberg_square_6x6", "heisenberg_chain_32_symm",
                                                     "heisenberg_chain_36_symm"])
    args = ap.parse_args()
    print("card:", card(), flush=True)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    for name in args.workloads:
        basis, matrix = load_config_from_yaml(os.path.join(ROOT, "data", name + ".yaml"))
        op = Operator(matrix)
        op.basis.build()
        n = op.basis.numberStates()
        op.use_torch_stream()
        print(f"== {name}: N={n}", flush=True)
        rng = np.random.default_rng(42)
        for dt in args.dtypes.split(","):
            cplx = dt == "c128"
            x = rng.random(n) - 0.5
            if cplx:
                x = x + 1j * (rng.random(n) - 0.5)
            xd = torch.from_numpy(x).cuda()
            yd = torch.zeros_like(xd)
            # (float64: two-slot buckets, 2 per state in both layouts)
            tables = ([] if args.no_hashed else [("hashed", 0, 14, 8, 0, 0, 0)]) + [
                (f"ordered D={d} b={b} l2={m}" + (f" W={w}" if m != "0" else ""), 1, int(d), int(b), int(m), int(w), 0)
                for d in args.bits.split(",") if d
                for b in (args.buckets.split(",") if cplx else ["2"])
                for m in args.l2.split(",")
                for w in (args.l2_window.split(",") if m != "0" else ["0"])] + [
                (f"dense D={d} l2={m}" + (f" W={w}" if m != "0" else ""), 1, int(d), 8, int(m), int(w), 1)
                for d in args.dense_bits.split(",")
                for m in args.l2.split(",") if args.dense_windows
                for w in (args.dense_windows.split(",") if m != "0" else ["0"])]
            ctas_list = [int(c) for c in args.ctas.split(",")]
            configs = [(c[0] + (f" ctas={k}" if len(ctas_list) > 1 else ""), *c[1:], k) for c in tables for k in ctas_list]
            times = {c[0]: [] for c in configs}
            worst = {c[0]: 0.0 for c in configs}
            ref = None
            placed = {}
            resident = {}
            for _ in range(args.rounds):
                for label, table, bits, buckets, l2, window, dense, ctas in configs:
                    op.set_option("rows_ctas", ctas)
                    op.set_option("rows_dense_order", dense)
                    op.set_option("rows_l2", l2)
                    op.set_option("rows_l2_window", window)
                    op.set_option("rows_table", table)
                    op.set_option("rows_table_bits", bits)
                    op.set_option("rows_table_buckets", buckets)
                    for _ in range(2):   # the first product rebuilds the table
                        op.matvec(xd, yd)
                    torch.cuda.synchronize()
                    assert op.info("rows") == 1, "k_rows does not apply"
                    assert op.info("rows_dense_order_on") == dense
                    resident[label] = op.info("rows_ctas_resident")
                    if dense and label not in placed:
                        placed[label] = op.info("rows_dense_order_placed")
                    for k in range(args.products):
                        flush.fill_(k)
                        s = torch.cuda.Event(enable_timing=True)
                        e = torch.cuda.Event(enable_timing=True)
                        s.record()
                        op.matvec(xd, yd)
                        e.record()
                        torch.cuda.synchronize()
                        times[label].append(s.elapsed_time(e))
                    op.synchronize()
                    if ref is None:
                        ref = yd.clone()
                    diff = (yd - ref).abs()
                    bound = torch.clamp(1e-12 * torch.maximum(yd.abs(), ref.abs()), min=1e-14)
                    bad = int((diff > bound).sum())
                    if bad:
                        raise SystemExit(f"{label}: {bad} elements differ from {configs[0][0]}")
                    worst[label] = max(worst[label], float(diff.max() / ref.abs().max()))
            base = float(np.median(times[configs[0][0]]))
            for label, *_ in configs:
                t = np.array(times[label])
                med = float(np.median(t))
                print(f"  {dt:4s} {label:30s} median {med:8.3f} ms  min {t.min():8.3f}  max {t.max():8.3f}  "
                      f"({len(t)} products)  vs first {100 * (med / base - 1):+6.1f} %  max rel diff {worst[label]:.1e}"
                      f"  resident CTAs/SM {resident[label]}"
                      + (f"  placed {placed[label]} of {n} ({n - placed[label]} left over)" if label in placed else ""),
                      flush=True)
        op.close()


if __name__ == "__main__":
    main()
