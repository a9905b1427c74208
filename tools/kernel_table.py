"""Markdown table for DESIGN.md §5e: every pass of the headline frame with its algorithmic bytes (bench.PASS_BYTES, SURVEY §8a), its measured time (a bench line),
the HBM roofline fraction that follows, and what ncu says bounds it (profiles/ncu_kernel_table.json, where present).   python tools/kernel_table.py <bench line>.json"""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import bench
b = json.loads(open(sys.argv[1]).read().strip().splitlines()[-1])
wl = b["config"]["workload"]; W, H = b["config"]["resolution"]; OW, OH = b["config"]["output_resolution"]
F, Hh, O = W * H, ((W + 1) // 2) * ((H + 1) // 2), OW * OH
peak = b["roofline"]["peak"]; pp = b["roofline"]["per_pass_ms"]
ncu = bench.load_ncu_table().get(wl, {})
print("| pass (rg label) | algorithmic bytes | per launch | ms | GB/s | % of HBM peak | ncu DRAM MB | issue-active % | occupancy % | lanes / inst | bound by |")
print("|---|---|---|---|---|---|---|---|---|---|---|")
for k, ms in sorted(pp.items(), key=lambda kv: -kv[1]):
    if k.startswith("tile "): continue
    kind, v = bench.PASS_BYTES[k]
    if kind == "F": unit = f"{v} B / render px"
    elif kind == "Hh": unit = f"{v} B / half-res px"
    elif kind == "const": unit = f"{v / 1e6:.1f} MB fixed" if v else "per live entry (count on the device)"
    else: unit = f"{v[0]} B / {'output' if kind.startswith('O') else 'render'} px + {v[1]} B / {'render' if kind.startswith('O') else 'half-res'} px"
    nb = bench.pass_bytes(k, F, Hh, O)
    n = ncu.get(k, {})
    gbs = nb / (ms * 1e-3) / 1e9 if nb else 0.0
    ia, occ, tpi = n.get("issue_active_pct"), n.get("occupancy_pct"), n.get("threads_per_inst")
    bound = "—"
    if ia is not None:
        bound = "instruction issue" if ia >= 65 else ("latency / divergence (ray traversal)" if (tpi or 32) < 20 else ("latency (grid too small)" if (occ or 100) < 30 else "issue + latency"))
    print(f"| {k} | {unit} | {nb / 1e6:.1f} MB | {ms:.3f} | {gbs:.0f} | {100 * gbs / peak:.1f} | " + (f"{n['dram_bytes'] / 1e6:.1f}" if n else "—") + " | " + (f"{ia:.0f}" if ia is not None else "—") + " | " + (f"{occ:.0f}" if occ is not None else "—") + " | " + (f"{tpi:.1f}" if tpi is not None else "—") + f" | {bound} |")
