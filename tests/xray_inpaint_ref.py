"""inpaint_xray_quadtree restated on the CPU with numpy, for the tests (xray/src/bin/inpaint_xray_quadtree.rs, xray/src/inpaint.rs):
the adjacent leaves, the stitch, the close, the nearest-sample fill (the project's replacement of texture synthesis: DESIGN.md
section 3), the f32 blends, the crop and assign_background_color, and the parents of create_non_leaf_nodes through
tests/xray_merge_ref.py's oracle.  Shares no code with csrc/.  Images are (rows, columns, 4) uint8 arrays, row 0 at the top;
spatial y grows upwards, so the Top neighbour (y + 1) lies above."""
import io
import os

import numpy as np

import xray_merge_ref as M

TRANSPARENT = np.array([255, 255, 255, 0], np.uint8)  # TRANSPARENT.to_u8() (src/color.rs:154)
DIRS = ((-1, 0), (0, 1), (1, 0), (0, -1))  # Left, Top, Right, Bottom


def xy(level, index):
    """SpatialNodeId::from(NodeId) (quadtree/src/lib.rs:313-331)."""
    x = y = 0
    for i in range(1, level + 1):
        mask, d = 1 << (level - i), index >> (2 * (level - i))
        if d & 1:
            y |= mask
        if d & 2:
            x |= mask
    return x, y


def index_of(level, x, y):
    """NodeId::from(SpatialNodeId) (lib.rs:333-351)."""
    idx = 0
    for i in range(1, level + 1):
        idx <<= 2
        mask = 1 << (level - i)
        idx += (1 if y & mask else 0) + (2 if x & mask else 0)
    return idx


def neighbor(level, index, dx, dy):
    """SpatialNodeId::neighbor (lib.rs:290-309), or None outside the level."""
    x, y = xy(level, index)
    x, y = x + dx, y + dy
    return index_of(level, x, y) if 0 <= x < (1 << level) and 0 <= y < (1 << level) else None


def adjacent(D, leaves, nbr_metas):
    """get_adjacent_leaf_node_ids (:41-71): nbr_metas[d] is the Meta of R's neighbour in DIRS[d], or None."""
    out = set()
    for (dx, dy), m in zip(DIRS, nbr_metas):
        if m is None:
            continue
        for (l, i) in m.nodes:
            if l != m.deepest or l != D:
                continue
            o = neighbor(D, i, -dx, -dy)
            if o is not None and o in leaves:
                out.add(i)
    return sorted(out)


# ---- per-image steps -------------------------------------------------------------------------------------------------------

def _window_count(a, k, axis):
    """Per pixel: the number of set pixels of `a` (bool) within distance k along `axis`, and the window's length, clipped."""
    n = a.shape[axis]
    c = np.cumsum(a.astype(np.int64), axis=axis)
    c = np.concatenate([np.zeros_like(np.take(c, [0], axis=axis)), c], axis=axis)
    p = np.arange(n)
    hi, lo = np.minimum(p + k, n - 1) + 1, np.maximum(p - k, 0)
    cnt = np.take(c, hi, axis=axis) - np.take(c, lo, axis=axis)
    shape = [1, 1]
    shape[axis] = n
    return cnt, (hi - lo).reshape(shape)


def close(mask, k):
    """close(mask, LInf, k): dilate (a pixel with alpha != 0 within the window), then erode (no unset pixel within it); only
    in-image pixels count."""
    d = _window_count(mask, k, 1)[0] > 0
    d = _window_count(d, k, 0)[0] > 0
    c1, l1 = _window_count(d, k, 1)
    e = c1 == l1
    c0, l0 = _window_count(e, k, 0)
    return c0 == l0


def near_rows(sample):
    """Column pass: the row of the nearest sample in each pixel's column, the upper on a tie; -1 when none."""
    h, w = sample.shape
    r = np.arange(h)[:, None]
    up = np.maximum.accumulate(np.where(sample, r, -1), axis=0)
    down = np.flipud(np.minimum.accumulate(np.flipud(np.where(sample, r, h * 4)), axis=0))
    use_down = (down < h) & ((up < 0) | (down - r < r - up))
    return np.where(use_down, down, up)


def nearest_sample(sample, holes):
    """For every hole pixel: the (row, column) of the nearest sample, the smaller column then the smaller row on a tie."""
    nr = near_rows(sample)
    hr, hc = np.nonzero(holes)
    if len(hr) == 0:
        return hr, hc, hr, hc
    w = sample.shape[1]
    g = np.where(nr >= 0, (np.arange(sample.shape[0])[:, None] - nr) ** 2, np.int64(1) << 60)
    out_c = np.empty(len(hr), np.int64)
    for s in range(0, len(hr), 4096):  # argmin takes the first, i.e. the smallest column
        rr, cc = hr[s:s + 4096], hc[s:s + 4096]
        val = (cc[:, None] - np.arange(w)[None, :]) ** 2 + g[rr]
        out_c[s:s + 4096] = np.argmin(val, axis=1)
    return hr, hc, nr[hr, out_c], out_c


def inpaint(img, k):
    """inpaint (inpaint.rs:24-44) with the nearest-sample fill.  Returns (image, hole pixels)."""
    alpha = img[:, :, 3] != 0
    holes = close(alpha, k) & ~alpha
    out = img.copy()
    hr, hc, sr, sc = nearest_sample(alpha, holes)
    out[hr, hc] = img[sr, sc]
    return out, int(holes.sum())


def round_away(v):
    """f32::round (half away from zero) of non-negative f32 values, as u8."""
    v = v.astype(np.float64)
    return np.clip(np.floor(v + 0.5), 0, 255).astype(np.uint8)


def blend(nb, cur, T, axis):
    """interpolate_subimages (utils.rs:47-83) of the neighbour's and the current image's halves (both (.., .., 4) uint8): the
    neighbour weighted i / (T - 1) along `axis` (1: columns, Right; 0: rows, Bottom), every product and sum in f32."""
    i = np.arange(nb.shape[axis], dtype=np.float32)
    wt = (i / np.float32(T - 1)).astype(np.float32)
    wt = wt[None, :, None] if axis == 1 else wt[:, None, None]
    one = np.float32(1.0)
    v = nb.astype(np.float32) * wt + cur.astype(np.float32) * (one - wt)
    return round_away(v.astype(np.float32))


def background(img, bg):
    """assign_background_color (generation.rs:686-707): alpha < 128 -> bg."""
    out = img.copy()
    out[img[:, :, 3] < 128] = np.array(bg, np.uint8)
    return out


def stitch(x, y, tiles, T):
    """stitched_image (inpaint.rs:90-121) of the leaf at (x, y): `tiles` maps (x, y) to the visible tiles."""
    w = T // 2
    out = np.empty((2 * T, 2 * T, 4), np.uint8)
    out[:] = TRANSPARENT
    for dy in (-1, 0, 1):  # image rows: -1 above (Top, y + 1)
        for dx in (-1, 0, 1):
            t = tiles.get((x + dx, y - dy))
            if t is None:
                continue
            r0, c0 = w + dy * T, w + dx * T
            rs, cs = max(r0, 0), max(c0, 0)
            re, ce = min(r0 + T, 2 * T), min(c0 + T, 2 * T)
            out[rs:re, cs:ce] = t[rs - r0:re - r0, cs - c0:ce - c0]
    return out


def inpaint_leaves(tiles, leaves, T, k, bg):
    """perform_inpainting then assign_background_color over `leaves` ((x, y) positions) from the visible `tiles`.  Returns
    ({(x, y): final T x T image}, hole pixels of the leaves' inpaint images)."""
    if k == 0:
        return {p: background(tiles[p], bg) for p in leaves}, 0
    imgs, holes = {}, 0
    for (x, y) in leaves:
        imgs[(x, y)], h = inpaint(stitch(x, y, tiles, T), k)
        holes += h
    for (x, y) in leaves:
        r = (x + 1, y)
        if r in imgs:
            v = blend(imgs[r][:, :T], imgs[(x, y)][:, T:], T, 1)
            imgs[r][:, :T] = v
            imgs[(x, y)][:, T:] = v
    for (x, y) in leaves:
        b = (x, y - 1)
        if b in imgs:
            v = blend(imgs[b][:T], imgs[(x, y)][T:], T, 0)
            imgs[b][:T] = v
            imgs[(x, y)][T:] = v
    w = T // 2
    return {p: background(im[w:w + T, w:w + T], bg) for p, im in imgs.items()}, holes


def meta_name(level, index):
    return "meta" + M.node_name(level, index)[1:] + ".pb"


def read_png(path):
    from PIL import Image

    return np.asarray(Image.open(io.BytesIO(open(path, "rb").read())).convert("RGBA"))


def inpaint_dir(input_dir, k, bg, root=(0, 0), in_place=False):
    """The whole of inpaint_xray_quadtree over `input_dir`: ({(level, index): image} of the leaves and the parents, adjacent
    leaf indices, hole pixels).  In place every <id>.png at the deepest level is visible, else the leaves and the adjacent
    leaves."""
    import oracle_api as O

    L, ri = root
    meta = M.read_meta(open(os.path.join(input_dir, meta_name(L, ri)), "rb").read())
    D, T = meta.deepest, meta.tile
    leaves = sorted(i for (l, i) in meta.nodes if l == D)
    nbr = []
    for dx, dy in DIRS:
        n = neighbor(L, ri, dx, dy)
        p = os.path.join(input_dir, meta_name(L, n)) if n is not None else None
        nbr.append(M.read_meta(open(p, "rb").read()) if p and os.path.exists(p) else None)
    adj = adjacent(D, set(leaves), nbr)
    if in_place:
        names = {f[:-4] for f in os.listdir(input_dir) if f.endswith(".png")}
        vis = [i for i in range(4 ** D) if M.node_name(D, i) in names] if D <= 6 else None
        assert vis is not None
    else:
        vis = sorted(set(leaves) | set(adj))
    tiles = {xy(D, i): read_png(os.path.join(input_dir, M.node_name(D, i) + ".png")) for i in vis}
    out, holes = inpaint_leaves(tiles, [xy(D, i) for i in leaves], T, k, bg)
    res = {(D, index_of(D, *p)): im for p, im in out.items()}
    cur = {(D, i) for i in leaves}
    for level in range(D - 1, L - 1, -1):
        cur = {(l - 1, i >> 2) for l, i in cur}
        for (l, i) in sorted(cur):
            ch = [res.get((l + 1, 4 * i + c)) for c in range(4)]
            res[(l, i)] = O.build_parent_tile(ch, bg, T)
    return res, adj, holes
