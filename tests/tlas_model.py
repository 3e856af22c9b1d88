"""numpy restatement of the ray caster's per-world TLAS build (kernels_render.cu), in
float32 where the kernels use float32.  renderBuildTLASKernel (worlds of up to 128
instances) and renderBuildLargeTLASKernel (above) both call one device function per rule,
named after each rule below:

  1. bounds of the instance box centres (centreBounds), 10-bit-per-axis Morton code of
     each centre, key = morton << 32 | gather index (mortonKey; keys are unique, so the
     sorted order is unique);
  2. Karras' split over the sorted keys, delta = -1 outside the world's segment
     (karrasSplit);
  3. bottom-up boxes (mergeBoxes; min / max: independent of the order nodes are finished in);
  4. breadth-first collapse to 4-wide nodes: a node starts with its binary children and
     repeatedly expands the inner child with the largest surface area (expandWide,
     wideChildArea; first maximum wins);
  5. quantizeNode (render_bvh.h) and the child encoding (writeWideNode).

build_tlas() returns the tree canonicalised depth-first from the root with children in
slot order, so it can be compared byte for byte with the engine's nodes after the same
canonicalisation (the engine numbers wide nodes in the order its threads reach them)."""
from __future__ import annotations

import numpy as np

F32 = np.float32
NODE_BYTES = 60
# traversal budget (kernels_render.cu): kTraceStack entries per ray, shared by the TLAS and
# the BLAS; a TLAS of wide depth D holds at most 3 * D entries when a BLAS starts, and the
# builder rejects trees deeper than kMaxTLASDepth so a BLAS always keeps kBLASStackReserve
TRACE_STACK = 48
BLAS_STACK_RESERVE = 12
MAX_TLAS_DEPTH = (TRACE_STACK - BLAS_STACK_RESERVE) // 3


def _expand_bits10(v):
    v = v.astype(np.uint64)
    v = (v * 0x00010001) & 0xFF0000FF
    v = (v * 0x00000101) & 0x0F00F00F
    v = (v * 0x00000011) & 0xC30C30C3
    v = (v * 0x00000005) & 0x49249249
    return v


def morton_keys(box_lo, box_hi):
    c = F32(0.5) * (box_lo + box_hi)
    lo, hi = c.min(axis=0), c.max(axis=0)
    ext = (hi - lo).astype(F32)
    code = np.zeros(len(c), dtype=np.uint64)
    for a in range(3):
        with np.errstate(divide="ignore", invalid="ignore"):
            u = np.where(ext[a] > 0, (c[:, a] - lo[a]) / ext[a], F32(0)).astype(F32)
        u = np.minimum(np.maximum(u * F32(1024), F32(0)), F32(1023))
        code |= _expand_bits10(u.astype(np.uint32)) << np.uint64(a)
    return (code << np.uint64(32)) | np.arange(len(c), dtype=np.uint64)


def _fma(a, b, c):
    # float32 fma through float64 (the product of two floats is exact there)
    return F32(np.float64(a) * np.float64(b) + np.float64(c))


def child_area(lo, hi):
    """wideChildArea(): dx*dy + dy*dz + dz*dx as the kernel evaluates it (fmas spelled out)."""
    dx, dy, dz = F32(hi[0] - lo[0]), F32(hi[1] - lo[1]), F32(hi[2] - lo[2])
    return _fma(dx, dz, _fma(dx, dy, F32(dy * dz)))


def quantize_node(cmin, cmax):
    """quantizeNode (render_bvh.h) -> 60 bytes with childrenIdx left 0xFFFFFFFF."""
    k = len(cmin)
    lo, hi = cmin.min(axis=0), cmax.max(axis=0)
    exps = np.zeros(3, dtype=np.int8)
    inv = np.zeros(3, dtype=F32)
    for a in range(3):
        extent = F32(hi[a] - lo[a])
        if extent > 0:
            e = int(np.ceil(np.log2(np.float64(F32(extent / F32(255))))))
        else:
            e = -126
        e = min(max(e, -126), 126)
        while e < 126 and np.ldexp(F32(255), e) < extent:
            e += 1
        exps[a] = e
        inv[a] = np.ldexp(F32(1), -e)
    q = np.zeros((2, 3, 4), dtype=np.uint8)       # [min / max][axis][child]
    for i in range(k):
        for a in range(3):
            ql = np.floor(F32((cmin[i, a] - lo[a]) * inv[a]))
            qh = np.ceil(F32((cmax[i, a] - lo[a]) * inv[a]))
            q[0, a, i] = np.uint8(min(max(ql, 0), 255))
            q[1, a, i] = np.uint8(min(max(qh, 0), 255))
    raw = bytearray(NODE_BYTES)
    raw[0:12] = lo.astype(F32).tobytes()
    raw[12:15] = exps.tobytes()
    raw[15] = k
    # triSize stays 0 (TLAS leaves are instances)
    raw[20:44] = q.reshape(-1).tobytes()
    raw[44:60] = b"\xff" * 16
    return raw


def _karras(skeys):
    n = len(skeys)
    keys = [int(k) for k in skeys]

    def delta(i, j):
        if j < 0 or j >= n:
            return -1
        return 64 - (keys[i] ^ keys[j]).bit_length()

    left = np.zeros(n - 1, dtype=np.int64)
    right = np.zeros(n - 1, dtype=np.int64)
    for i in range(n - 1):
        d = 1 if delta(i, i + 1) - delta(i, i - 1) >= 0 else -1
        dmin = delta(i, i - d)
        lmax = 2
        while delta(i, i + lmax * d) > dmin:
            lmax <<= 1
        l, t = 0, lmax >> 1
        while t >= 1:
            if delta(i, i + (l + t) * d) > dmin:
                l += t
            t >>= 1
        j = i + l * d
        dnode = delta(i, j)
        s, t = 0, (l + 1) >> 1
        while True:
            if delta(i, i + (s + t) * d) > dnode:
                s += t
            if t == 1:
                break
            t = (t + 1) >> 1
        gamma = i + s * d + min(d, 0)
        first, last = min(i, j), max(i, j)
        left[i] = ~gamma if first == gamma else gamma          # < 0: ~leaf (sorted position)
        right[i] = ~(gamma + 1) if last == gamma + 1 else gamma + 1
    return left, right


def build_tlas(box_lo, box_hi):
    """-> (canonical node bytes [nodes, 60] uint8, wide depth).  box_lo / box_hi: float32 [n, 3]."""
    box_lo = np.asarray(box_lo, dtype=F32)
    box_hi = np.asarray(box_hi, dtype=F32)
    n = len(box_lo)
    if n == 0:
        return np.zeros((0, NODE_BYTES), dtype=np.uint8), 0
    keys = morton_keys(box_lo, box_hi)
    order = np.argsort(keys, kind="stable")
    if n == 1:
        raw = quantize_node(box_lo[:1], box_hi[:1])
        raw[16] = 0
        raw[44:48] = np.uint32(0x80000000).tobytes()
        return np.frombuffer(bytes(raw), dtype=np.uint8).reshape(1, NODE_BYTES).copy(), 1
    left, right = _karras(keys[order])
    leaf_lo, leaf_hi = box_lo[order], box_hi[order]
    node_lo = np.zeros((n - 1, 3), dtype=F32)
    node_hi = np.zeros((n - 1, 3), dtype=F32)

    def box(c):
        return (node_lo[c], node_hi[c]) if c >= 0 else (leaf_lo[~c], leaf_hi[~c])

    # post-order over the binary tree without recursion
    stack, done = [0], np.zeros(n - 1, dtype=bool)
    while stack:
        x = stack[-1]
        pending = [c for c in (left[x], right[x]) if c >= 0 and not done[c]]
        if pending:
            stack.extend(pending)
            continue
        stack.pop()
        (al, ah), (bl, bh) = box(left[x]), box(right[x])
        node_lo[x] = np.minimum(al, bl)
        node_hi[x] = np.maximum(ah, bh)
        done[x] = True

    def wide_children(b):
        kids = [int(left[b]), int(right[b])]
        while len(kids) < 4:
            pick, best = -1, F32(-1)
            for c, k in enumerate(kids):
                if k < 0:
                    continue
                area = child_area(node_lo[k], node_hi[k])
                if area > best:
                    best, pick = area, c
            if pick < 0:
                break
            inner = kids[pick]
            kids[pick] = int(left[inner])
            kids.append(int(right[inner]))
        return kids

    # depth first, children in slot order: canonical numbering
    out, depth = [], 0
    todo = [(0, 1, None, None)]        # (binary node, depth, parent canonical index, slot)
    while todo:
        b, dep, parent, slot = todo.pop()
        me = len(out)
        depth = max(depth, dep)
        if parent is not None:
            out[parent][44 + 4 * slot:48 + 4 * slot] = np.uint32(me).tobytes()
        kids = wide_children(b)
        cmin = np.array([box(k)[0] for k in kids], dtype=F32)
        cmax = np.array([box(k)[1] for k in kids], dtype=F32)
        raw = quantize_node(cmin, cmax)
        for c, k in enumerate(kids):
            if k < 0:
                raw[44 + 4 * c:48 + 4 * c] = np.uint32(0x80000000 | int(order[~k])).tobytes()
        out.append(raw)
        for c in reversed(range(len(kids))):
            if kids[c] >= 0:
                todo.append((kids[c], dep + 1, me, c))
    return np.frombuffer(b"".join(bytes(r) for r in out), dtype=np.uint8).reshape(-1, NODE_BYTES).copy(), depth


def canonicalise(nodes_raw):
    """Engine nodes of one world (uint8 [count, 60]) -> depth-first canonical form."""
    nodes_raw = np.asarray(nodes_raw, dtype=np.uint8)
    if len(nodes_raw) == 0:
        return nodes_raw.copy()
    children = nodes_raw[:, 44:60].copy().view(np.uint32)
    out, todo = [], [(0, None, None)]
    while todo:
        g, parent, slot = todo.pop()
        me = len(out)
        if parent is not None:
            out[parent][44 + 4 * slot:48 + 4 * slot] = np.uint32(me).tobytes()
        out.append(bytearray(nodes_raw[g].tobytes()))
        for c in reversed(range(4)):
            ch = int(children[g, c])
            if ch != 0xFFFFFFFF and not ch & 0x80000000:
                todo.append((ch, me, c))
    return np.frombuffer(b"".join(bytes(r) for r in out), dtype=np.uint8).reshape(-1, NODE_BYTES).copy()


def same_tree(a, b):
    """Byte equality of two canonical trees, with -0.0 and +0.0 taken as the same minPoint."""
    if a.shape != b.shape:
        return False
    if len(a) == 0:
        return True
    pa = a[:, 0:12].copy().view(F32) + F32(0)
    pb = b[:, 0:12].copy().view(F32) + F32(0)
    return bool(np.array_equal(pa, pb) and np.array_equal(a[:, 12:], b[:, 12:]))


def decode(nodes):
    n = len(nodes)
    return dict(
        min_point=nodes[:, 0:12].copy().view(F32).reshape(n, 3),
        exp=nodes[:, 12:15].copy().view(np.int8).reshape(n, 3),
        num_children=nodes[:, 15],
        qmin=np.stack([nodes[:, 20:24], nodes[:, 24:28], nodes[:, 28:32]], axis=2),
        qmax=np.stack([nodes[:, 32:36], nodes[:, 36:40], nodes[:, 40:44]], axis=2),
        children=nodes[:, 44:60].copy().view(np.uint32).reshape(n, 4),
    )
