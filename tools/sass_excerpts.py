"""profiles/r02_sass_excerpts.txt: which of our kernels contain TMA-engine copies (UBLKCP = cp.async.bulk), transaction
barriers (SYNCS.*) and warp shuffles (SHFL.*) — from `cuobjdump -sass` of the shipping objects (no GPU needed).   python tools/sass_excerpts.py"""
import subprocess, re, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
objs = ['kjb_passes_taa.cu.o', 'kjb_passes_rtdgi.cu.o', 'kjb_passes_rtr.cu.o', 'kjb_passes_ircache.cu.o', 'kjb_api.cu.o']
out = ["# SASS evidence (cuobjdump -sass of kajiya_b200/csrc/_obj/*.o, sm_90a, the shipping build): TMA-engine copies (UBLKCP = cp.async.bulk),",
       "# transaction barriers (SYNCS.*), warp shuffles (SHFL.*) per kernel: instruction counts and one line per distinct form.  Regenerate: python tools/sass_excerpts.py", ""]
pat = re.compile(r'UBLKCP|SYNCS\.|SHFL\.|ELECT')
for o in objs:
    txt = subprocess.run(['cuobjdump', '-sass', os.path.join(ROOT, 'kajiya_b200/csrc/_obj', o)], stdout=subprocess.PIPE, text=True).stdout
    fn, hits = None, {}
    for line in txt.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            fn = m.group(1); continue
        if fn and pat.search(line) and '/*' in line:
            hits.setdefault(fn, []).append(line.split('*/', 1)[1].split('/*')[0].strip().rstrip(';').strip())
    for fn, l in hits.items():
        name = subprocess.run(['c++filt', fn], stdout=subprocess.PIPE, text=True).stdout.strip().split('(')[0]
        kinds = {}
        for ins in l:
            k = ins.split()[0] if not ins.startswith('@') else ins.split()[1]
            kinds[k] = kinds.get(k, 0) + 1
        out.append(f"{o[:-5]} :: {name}")
        out.append("    counts: " + ", ".join(f"{k} x{v}" for k, v in sorted(kinds.items())))
        seen = set()
        for ins in l:
            k = re.sub(r'\s+', ' ', ins); key = k.split('[')[0]
            if key not in seen:
                seen.add(key); out.append("    " + k)
        out.append("")
open(os.path.join(ROOT, 'profiles', 'r02_sass_excerpts.txt'), 'w').write("\n".join(out))
print(len(out), "lines")
