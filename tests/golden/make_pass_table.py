"""Extracts the render-graph pass declarations of the hot path from kajiya's Rust sources — mechanically, so that the table is independent
of this repo's C++ host mirror — into tests/golden/pass_table.json.  Run against a checkout of kajiya:

    python tests/golden/make_pass_table.py <path to the kajiya checkout>

For every `SimpleRenderPass::new_compute / new_rt(rg.add_pass("label"), shader...)` builder chain the table records, in call order, the
binding methods (`read`, `read_aspect`, `write`, `write_no_sync`, `constants`, `bind`, `bind_mut`, `raw_descriptor_set`, ...) with their
argument text, and the terminal call (`dispatch`, `dispatch_indirect`, `trace_rays`, `trace_rays_indirect`).  Binding index = call order
(crates/lib/kajiya-rg/src/hl.rs:266,324,354-359).  It also records the order in which the irradiance cache's `bind_mut` binds its buffers.
tests/test_host_mirror.py asserts kjb_world.cpp against it."""
import json, os, re, sys

REF = sys.argv[1]
FILES = ["crates/lib/kajiya/src/renderers/rtdgi.rs", "crates/lib/kajiya/src/renderers/ircache.rs", "crates/lib/kajiya/src/renderers/rtr.rs",
         "crates/lib/kajiya/src/renderers/taa.rs", "crates/lib/kajiya/src/renderers/reprojection.rs", "crates/lib/kajiya/src/renderers/half_res.rs",
         "crates/lib/kajiya/src/renderers/ssgi.rs", "crates/lib/kajiya/src/renderers/lighting.rs", "crates/lib/kajiya/src/renderers/shadow_denoise.rs",
         "crates/lib/kajiya/src/renderers/deferred.rs", "crates/lib/kajiya/src/renderers/shadows.rs", "crates/lib/kajiya/src/renderers/prefix_scan.rs",
         "crates/lib/kajiya/src/renderers/reference.rs", "crates/lib/kajiya/src/renderers/sky.rs"]
TERMINALS = {"dispatch", "dispatch_indirect", "trace_rays", "trace_rays_indirect"}


def balanced(src, i):
    """src[i] == '(' -> index just past the matching ')' (string literals skipped)"""
    depth = 0
    while i < len(src):
        c = src[i]
        if c == '"':
            i += 1
            while src[i] != '"':
                i += 2 if src[i] == "\\" else 1
        elif c in "([{":
            depth += 1
        elif c in ")]}":
            depth -= 1
            if depth == 0:
                return i + 1
        i += 1
    raise ValueError("unbalanced")


def squash(s):
    return re.sub(r"\s+", " ", s).strip()


def passes_of(path):
    src = open(os.path.join(REF, path)).read()
    src_nc = re.sub(r"//[^\n]*", lambda m: " " * len(m.group(0)), src)   # comments blanked, offsets kept
    out = []
    for m in re.finditer(r"SimpleRenderPass::new_(compute_rust|compute|rt)\s*\(", src_nc):
        kind = m.group(1)
        end = balanced(src_nc, m.end() - 1)
        head = squash(src_nc[m.end():end - 1])
        lab = re.search(r'add_pass\(\s*"([^"]+)"', head)
        label = lab.group(1) if lab else None
        shaders = re.findall(r'"(/shaders/[^"]+)"', head)
        calls, i, terminal = [], end, None
        while True:
            mm = re.match(r"\s*\.\s*([a-z_]+)\s*\(", src_nc[i:])
            if not mm:
                break
            a0 = i + mm.end() - 1
            a1 = balanced(src_nc, a0)
            name, arg = mm.group(1), squash(src_nc[a0 + 1:a1 - 1])
            i = a1
            if name in TERMINALS:
                terminal = {"m": name, "arg": arg}
                break
            calls.append({"m": name, "arg": arg})
        out.append({"file": path, "line": src.count("\n", 0, m.start()) + 1, "label": label, "label_expr": None if label else head.split(",")[0], "kind": kind,
                    "shaders": shaders, "calls": calls, "terminal": terminal})
    return out


def ircache_bind_mut_order():
    """buffer fields in the order `BindMutToSimpleRenderPass for IrcacheRenderState` (ircache.rs) binds them"""
    src = open(os.path.join(REF, "crates/lib/kajiya/src/renderers/ircache.rs")).read()
    body = src[src.index("impl<'rg, RgPipelineHandle> BindMutToSimpleRenderPass"):]
    body = body[:body.index("\n}\n")]
    return re.findall(r"(?:write_no_sync|read)\(&(?:mut )?self\.(\w+)\)", body)


table = []
for f in FILES:
    if os.path.exists(os.path.join(REF, f)):
        table += passes_of(f)
dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pass_table.json")
json.dump({"source": "EmbarkStudios/kajiya @ 9fdec0f, crates/lib/kajiya/src/renderers/*.rs", "generator": "tests/golden/make_pass_table.py", "passes": table,
           "ircache_bind_mut_order": ircache_bind_mut_order()}, open(dst, "w"), indent=1)
print(len(table), "passes ->", dst)
for p in table:
    print(f'{p["file"].split("/")[-1]}:{p["line"]:<4} {p["label"] or p["label_expr"]!s:32} {len(p["calls"]):2} calls  {p["terminal"]["m"] if p["terminal"] else "?"}')
