"""Cuts a small glTF out of a reference asset too large to store whole, for tests/test_asset.py:

    python tests/golden/make_reference_subsets.py <path to the kajiya checkout>

  reference_assets/meshes/conference_jake/  <- assets/meshes/conference: the "Cube" node (mesh 1) that carries the JPEG texture jake.jpg
                                               as base colour and emissive map, with the scene's full material, texture and sampler
                                               tables; the 35 MB buffer is cut down to that mesh's accessors."""
import json, os, shutil, sys

SRC = os.path.join(sys.argv[1], "assets", "meshes", "conference")
DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_assets", "meshes", "conference_jake")

g = json.load(open(os.path.join(SRC, "scene.gltf")))
blob = open(os.path.join(SRC, g["buffers"][0]["uri"]), "rb").read()
node = next(n for n in g["nodes"] if n["name"] == "Cube")
mesh = g["meshes"][node["mesh"]]
out_bin, views, accessors, remap = bytearray(), [], [], {}


def take(ai):
    if ai not in remap:
        acc = dict(g["accessors"][ai]); bv = g["bufferViews"][acc["bufferView"]]
        while len(out_bin) % 4:
            out_bin.append(0)
        nv = dict(bv, byteOffset=len(out_bin)); out_bin.extend(blob[bv.get("byteOffset", 0):bv.get("byteOffset", 0) + bv["byteLength"]])
        views.append(nv); acc["bufferView"] = len(views) - 1
        accessors.append(acc); remap[ai] = len(accessors) - 1
    return remap[ai]


prims = []
for p in mesh["primitives"]:
    q = dict(p, attributes={k: take(v) for k, v in p["attributes"].items()})
    if "indices" in q:
        q["indices"] = take(p["indices"])
    prims.append(q)
out = dict(g, scene=0, scenes=[{"name": "Scene", "nodes": [0]}], nodes=[dict(node, mesh=0)], meshes=[dict(mesh, primitives=prims)],
           accessors=accessors, bufferViews=views, buffers=[{"byteLength": len(out_bin), "uri": "scene.bin"}])
os.makedirs(DST, exist_ok=True)
json.dump(out, open(os.path.join(DST, "scene.gltf"), "w"), indent=1)
open(os.path.join(DST, "scene.bin"), "wb").write(bytes(out_bin))
for f in ("jake.jpg", "license.txt"):
    shutil.copyfile(os.path.join(SRC, f), os.path.join(DST, f))
print(DST, len(out_bin), "bytes of buffer")
