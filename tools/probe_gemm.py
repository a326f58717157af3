#!/usr/bin/env python
"""GPU probe: the batched GEMM alone, mean device time per launch, accuracy, the modelled HBM operand traffic of two
tile orders: the m-tile-fastest order of the first kernel versions and the grouped order the launcher picks now (the
same rule as pick_tile_order in csrc/gemm_tf32x3.cu, restated here), and the operand bytes the launch moves from the L2
into shared memory, with and without the A multicast of the CTA pairs, with the rate the measured time gives.  The
paired feed is also given for each output-tile width.

Every case is timed at each output-tile width the exact-B forms have (--tile-n 128 168 192 by default), the widths
alternated inside one call, with the shared-memory model of each width: bytes
written by TMA and read by the MMAs per tensor-core clock at peak rate, against about 128 B/clk of shared-memory
bandwidth per SM (DESIGN.md section 4.1).  The outputs of all widths must be bit-identical.

The kernel runs in clusters of 2 CTAs: a pair's work item is an m-tile and two adjacent n-tiles (an n-pair), so the
tile order is over m-tiles x n-pairs, a B panel is 256 rows, and the grid of the order is the number of pairs that
run at once (taken here as half the SMs; the launcher asks the device).

    python tools/probe_gemm.py [--precision f16x2|tf32x3|tf32x3-general] [--tile-n W ...] [--rounds R] [case ...]

--precision (default f16x2) is passed to Engine.gemm_abt.  f16x2 runs the exact-B fp16 form; tf32x3 runs the exact-B
tf32 form (B holds integer counts); tf32x3-general runs the 3-pass form, which has 128-column tiles only.

Cases: c2-shaped problems, a 4 096-row problem, the c3 shapes at full SK (8 100 packed rows: factor operand larger
than the L2) and the same c3 shapes with 1 024 rows (factor operand resident in the L2)."""
import argparse, json, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cnmf_b200.engine import Engine

BM = BN = 128            # output tile of the HBM tile-order model
KB_BYTES = 128           # bytes of one operand piece per row and k-block: 64 fp16 or 32 tf32 elements


def slices(Kd, splits, f16):
    """k-blocks per split-K slice, as the launcher partitions them (f16 slices start on even k-blocks)."""
    total_kb = -(-Kd // (64 if f16 else 32))
    splits = max(1, min(splits, total_kb))
    kbps = -(-total_kb // splits)
    if f16:
        kbps += kbps & 1
    return [min(kbps, total_kb - z * kbps) for z in range(-(-total_kb // kbps))]


def order_bytes(q_tiles, p_tiles, q_panel, p_panel, group, grid, budget):
    """Operand bytes one slice reads from HBM when groups of `group` panels of one operand (q) each sweep every panel of
    the other (p): the group is read once if it fits the L2 budget, else once per wave of the grid that passes over it;
    each p panel is read once per group."""
    if group * q_panel <= budget:
        q_reads = 1
    else:
        q_reads = min(p_tiles, -(-group * p_tiles // grid))
    return q_tiles * q_panel * q_reads + -(-q_tiles // group) * p_tiles * p_panel


def pick_order(m_tiles, n_tiles, a_panel, b_panel, grid, budget):
    """(bytes, group, group_n) of the cheapest grouped order; ties keep the m-tile-fastest order (group = m_tiles)."""
    best = None
    for group_n, q, p, qb, pb in ((0, m_tiles, n_tiles, a_panel, b_panel), (1, n_tiles, m_tiles, b_panel, a_panel)):
        for ng in range(1, q + 1):
            g = -(-q // ng)
            if ng > 1 and g == -(-q // (ng - 1)):
                continue
            b = order_bytes(q, p, qb, pb, g, grid, budget)
            if best is None or b < best[0]:
                best = (b, g, group_n)
    return best


def model(M, N, Kd, splits, l2, sms, f16, b_pieces):
    """Modelled operand bytes of the launch in both orders, and its L2 -> shared memory operand bytes.  A is two pieces;
    B is one exact operand (b_pieces = 1: fp16, or tf32 integer counts) or two tf32 pieces (the 3-pass form)."""
    m_tiles, n_tiles = -(-M // BM), -(-N // BN)
    n_pairs = -(-n_tiles // 2)
    kbs = slices(Kd, splits, f16)
    items = m_tiles * n_pairs * len(kbs)
    grid = min(items, sms // 2)
    budget = l2 // 2
    a_panel, b_panel = (BM * kbs[0] * KB_BYTES * 2, 2 * BN * kbs[0] * KB_BYTES * b_pieces)
    _, g, gn = pick_order(m_tiles, n_pairs, a_panel, b_panel, grid, budget)
    flat = grouped = 0
    for kb in kbs:
        ap, bp = BM * kb * KB_BYTES * 2, 2 * BN * kb * KB_BYTES * b_pieces
        flat += order_bytes(m_tiles, n_pairs, ap, bp, m_tiles, grid, budget)
        grouped += (order_bytes(n_pairs, m_tiles, bp, ap, g, grid, budget) if gn else
                    order_bytes(m_tiles, n_pairs, ap, bp, g, grid, budget))
    minimum = sum(m_tiles * BM * kb * KB_BYTES * 2 + n_tiles * BN * kb * KB_BYTES * b_pieces for kb in kbs)
    # L2 -> SM: every CTA loads its B tile each k-block; A (16 KB per piece and tile k-block) once per CTA unpaired,
    # once per pair with the multicast (each CTA of the pair loads half and receives the other half).
    piece = BM * KB_BYTES
    kb_total = sum(kbs)
    unpaired = m_tiles * n_tiles * kb_total * piece * (2 + b_pieces)
    paired = paired_feed(M, N, kb_total, BN, b_pieces)
    return {"m_fastest_GB": round(flat / 1e9, 3), "grouped_GB": round(grouped / 1e9, 3), "min_GB": round(minimum / 1e9, 3),
            "grouped_order": "%d %s per group" % (g, "n-pairs" if gn else "m-tiles"), "slices": len(kbs),
            "l2_to_smem_unpaired_GB": round(unpaired / 1e9, 2), "l2_to_smem_paired_GB": round(paired / 1e9, 2),
            "l2_to_smem_paired_GB_by_tile_n": {bn: round(paired_feed(M, N, kb_total, bn, b_pieces) / 1e9, 2)
                                               for bn in (128, 168, 192)}}


def smem_bytes_per_clock(bn):
    """Shared-memory bytes per tensor-core clock at peak rate, one k-block of a 128 x bn tile in an exact-B form: TMA
    writes both A pieces (128 rows) and B (bn rows) at 128 B a row; each of the 2 consumer warpgroups issues 8 MMAs
    (4 k-steps x 2 pieces), each reading its 2 KB A slice and a 32 B slice of all bn B rows; an m64 x bn MMA takes
    bn / 2 tensor clocks (f16 k16 and tf32 k8 alike).  (32 KB + 128 bn + 16 (2 KB + 32 bn)) / 8 bn = 8192 / bn + 80."""
    written = 2 * BM * KB_BYTES + bn * KB_BYTES
    read = 16 * (2048 + 32 * bn)
    return (written + read) / (8 * bn)


def paired_feed(M, N, kb_total, bn, b_pieces):
    """L2 -> shared memory operand bytes of a paired launch with 128 x bn tiles: per m-tile and k-block, the 128 rows of
    both A pieces once per pair (each CTA loads half and multicasts it) and every CTA's own bn-row B pieces.  Per FLOP
    that is 32 KB per 128 x 128 tile, 37 KB per 128 x 168 and 40 KB per 128 x 192 (f16x2): 12-17 % less when wider,
    before padding."""
    m_tiles, n_tiles = -(-M // BM), -(-(-(-N // 32) * 32) // bn)
    n_pairs = -(-n_tiles // 2)
    return m_tiles * kb_total * KB_BYTES * (2 * BM * n_pairs + b_pieces * bn * n_tiles)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--precision", choices=("f16x2", "tf32x3", "tf32x3-general"), default="f16x2")
    ap.add_argument("--tile-n", type=int, nargs="+", default=[128, 168, 192], help="forced output-tile widths")
    ap.add_argument("--rounds", type=int, default=3, help="timed calls per width, the widths alternated")
    ap.add_argument("cases", nargs="*", help="case names to run (default: all)")
    args = ap.parse_args()
    f16 = args.precision == "f16x2"
    import torch
    props = torch.cuda.get_device_properties(0)
    l2, sms = props.L2_cache_size, props.multi_processor_count
    eng = Engine(0)
    rng = np.random.RandomState(0)
    widths = [128] if args.precision == "tf32x3-general" else args.tile_n
    out = {"device": props.name, "l2_bytes": l2, "sms": sms, "precision": args.precision,
           "smem_B_per_clk": {"128x%d" % bn: round(smem_bytes_per_clock(bn), 1) for bn in (128, 168, 192)}}
    print("smem bytes per tensor clock at peak", json.dumps(out["smem_B_per_clk"]), flush=True)
    cases = {"c2_W_half": (1000, 20000, 2000, 1), "c2_H_half": (1000, 2000, 20000, 5),
             "mid_W_half": (4096, 16384, 2000, 1), "mid_H_half": (4096, 2000, 16384, 4),
             "tail_H_half": (128, 2000, 20000, 5), "tail_W_half": (128, 20000, 2000, 1),
             "c3_W_half_full": (8100, 50000, 2000, 1), "c3_H_half_full": (8100, 2000, 50000, 13),
             "c3_W_half_1024": (1024, 50000, 2000, 1), "c3_H_half_1024": (1024, 2000, 50000, 13)}
    only = args.cases
    for name, (M, N, K, sp) in cases.items():
        if only and name not in only:
            continue
        if M * K > 10 ** 8 or N * K > 10 ** 8:      # c3 sizes: float32 draws directly (the float64 ones need 3+ GB)
            g = np.random.default_rng(0)
            A = g.random((M, K), dtype=np.float32)
            B = g.poisson(1.5, size=(N, K)).astype(np.float32)
        else:
            A = np.abs(rng.standard_normal((M, K))).astype(np.float32)
            B = rng.poisson(1.5, size=(N, K)).astype(np.float32)
        b_exact = args.precision == "tf32x3"
        times = {w: [] for w in widths}
        C = None
        for _ in range(args.rounds):
            for w in widths:
                Cw, ms_w = eng.gemm_abt(A, B, precision=args.precision, splits=sp, reps=20, b_exact=b_exact, tile_n=w)
                times[w].append(ms_w)
                if C is None:
                    C = Cw
                elif not np.array_equal(Cw, C):
                    raise SystemExit("%s: tile_n=%d changed the result" % (name, w))
                del Cw
        ms = min(times[widths[0]])
        ref = A[:64].astype(np.float64) @ B.astype(np.float64).T
        err = float(np.linalg.norm(C[:64] - ref) / np.linalg.norm(ref))
        tail = A[-64:].astype(np.float64) @ B.astype(np.float64).T
        err2 = float(np.linalg.norm(C[-64:] - tail) / np.linalg.norm(tail))
        mdl = model(M, N, K, sp, l2, sms, f16, 1 if b_exact or f16 else 2)
        out[name] = {"shape": [M, N, K, sp], "ms": round(ms, 4), "tflops": round(2.0 * M * N * K / (ms * 1e-3) / 1e12, 1),
                     "l2_to_smem_TBps": round(mdl["l2_to_smem_paired_GB"] / ms, 2),
                     "rel_err_first_rows": err, "rel_err_last_rows": err2, "model": mdl,
                     "ms_by_tile_n": {w: [round(t, 4) for t in ts] for w, ts in times.items()},
                     "best_ms_by_tile_n": {w: round(min(ts), 4) for w, ts in times.items()}}
        print(name, json.dumps(out[name]), flush=True)
        del A, B, C
    print(json.dumps(out))


if __name__ == "__main__":
    main()
