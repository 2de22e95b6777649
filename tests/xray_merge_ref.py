"""merge_xray_quadtrees restated on the CPU, for the tests (xray/src/bin/merge_xray_quadtrees.rs): the meta files read with
python-protobuf (tests/proto_meta.py), the PNGs with Pillow, the checks of validate_and_merge_metadata, the rect from
Node::parent, the parents of create_non_leaf_nodes built level by level with the oracle's build_parent + Lanczos3
(oracle/oracle_xray_pyramid.hpp through oracle_api.build_parent_tile).  Shares no code with csrc/."""
import io
import os

import numpy as np

OK, INVALID, NOT_FOUND = 0, -1, -4


class Meta:
    def __init__(self, nodes, deepest=6, tile=256, rect=(0.0, 0.0, 64.0)):
        self.nodes, self.deepest, self.tile, self.rect = list(nodes), deepest, tile, rect


def read_meta(data):
    """Meta::from_proto (xray/src/lib.rs:59-116) of a version 2 or 3 meta file."""
    from proto_meta import XrayMeta

    m = XrayMeta.FromString(data)
    assert m.version in (2, 3), m.version
    r = m.bounding_rect
    rect = (r.min.x, r.min.y, r.edge_length) if r.HasField("min") else (r.deprecated_min.x, r.deprecated_min.y, r.deprecated_edge_length)
    return Meta([(n.level & 0xFF, n.index) for n in m.nodes], m.deepest_level & 0xFF, m.tile_size, rect)


def plan(metas):
    """validate_and_merge_metadata (:125-176) and the parents of create_non_leaf_nodes (generation.rs:656-682).  Returns (code,
    message) or (OK, (root level, deepest, tile, rect, sorted roots, set of parents, sorted merged nodes))."""
    if not metas:
        return NOT_FOUND, "No subquadtrees meta files found."
    roots = [(min(m.nodes), m) for m in metas if m.nodes]
    if not roots:
        return INVALID, "All subquadtress are empty."
    ids = [r for r, _ in roots]
    if len(set(ids)) != len(ids):
        return INVALID, "Not all roots are unique."
    if len({l for l, _ in ids}) != 1:
        return INVALID, "Not all roots have the same level."
    if len({m.deepest for m in metas}) != 1:
        return INVALID, "Not all meta files have the same deepest level."
    if len({m.tile for m in metas}) != 1:
        return INVALID, "Not all meta files have the same tile size."
    (level, index), m0 = roots[0]
    x, y, e = m0.rect
    while level > 0:  # Node::parent (quadtree/src/lib.rs:100-120)
        ci = index & 3
        if ci & 1:
            y -= e
        if ci & 2:
            x -= e
        e *= 2.0
        level, index = level - 1, index >> 2
    L = ids[0][0]
    cur, parents = set(ids), set()
    for _ in range(L):
        cur = {(l - 1, i >> 2) for l, i in cur}
        parents |= cur
    nodes = set(parents)
    for m in metas:
        nodes |= set(m.nodes)
    return OK, (L, metas[0].deepest, metas[0].tile, (x, y, e), sorted(ids), parents, sorted(nodes))


def node_name(level, index):
    return "r" + "".join(str((index >> (2 * l)) & 3) for l in range(level - 1, -1, -1))


def merge(input_dirs, background):
    """The merge of the sub-root builds in `input_dirs`: (meta as plan() returns it, {(level, index): RGBA array} of the
    parents).  The copied images are the input files themselves; the sub-roots are read from them."""
    from PIL import Image

    import oracle_api as O

    metas, pngs = [], {}
    for d in input_dirs:
        for name in sorted(os.listdir(d)):
            path = os.path.join(d, name)
            if os.path.isdir(path):
                continue
            if name.startswith("meta") and name.endswith(".pb"):
                metas.append(read_meta(open(path, "rb").read()))
            elif name.endswith(".png"):
                pngs[name] = path
    code, p = plan(metas)
    assert code == OK, p
    L, _, T, _, roots, parents, _ = p
    tiles = {r: np.asarray(Image.open(io.BytesIO(open(pngs[node_name(*r) + ".png"], "rb").read())).convert("RGBA")) for r in roots}
    out = {}
    for level in range(L - 1, -1, -1):
        for (l, i) in sorted(q for q in parents if q[0] == level):
            ch = [tiles.get((l + 1, 4 * i + k)) for k in range(4)]
            out[(l, i)] = tiles[(l, i)] = O.build_parent_tile(ch, background, T)
    return p, out
