"""Dev tool: dump and validate the per-world TLAS of the gallery fixture."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from sims import make_executor
from test_render_bvh import _decode_nodes

W, P = 2, 100
ex = make_executor("gallery", W, num_props=P, seed=5, resolution=16, rgbd=True)
step = ex.buildLaunchGraphAllTaskGraphs()
ex.run(step)
nodes_raw, ncount, inst_raw, icount, offsets = ex.renderDebugStructures()
print("instance counts", icount, "offsets", offsets, "tlas node counts", ncount)
for w in range(W):
    n = int(icount[w]); k = int(ncount[w]); o = int(offsets[w])
    inst = inst_raw[o:o + n].copy().view(np.float32).reshape(n, 19)
    lo_i, hi_i = inst[:, 13:16], inst[:, 16:19]
    nodes = _decode_nodes(nodes_raw[o:o + k])
    seen = np.zeros(n, dtype=int)
    stack = [0]; visited = 0; bad = 0
    while stack and visited < 4 * max(k, 1):
        g = stack.pop(); visited += 1
        scale = np.ldexp(1.0, nodes["exp"][g].astype(np.int32))
        for c in range(4):
            child = int(nodes["children"][g, c])
            if child == 0xFFFFFFFF: continue
            lo = nodes["min_point"][g] + scale * nodes["qmin"][g, c]
            hi = nodes["min_point"][g] + scale * nodes["qmax"][g, c]
            if child & 0x80000000:
                i = child & 0x7FFFFFFF
                if i >= n: print("leaf out of range", i); bad += 1; continue
                seen[i] += 1
                if not ((lo_i[i] >= lo - 1e-4).all() and (hi_i[i] <= hi + 1e-4).all()):
                    bad += 1
                    if bad < 5: print("leaf", i, "box", lo_i[i], hi_i[i], "not inside", lo, hi)
            else:
                if child >= k: print("child out of range", child, k); bad += 1; continue
                stack.append(child)
    print("world", w, "visited", visited, "of", k, "seen once:", (seen == 1).sum(), "of", n, "bad", bad)
    print("  root node", {a: nodes[a][0] for a in nodes})
    print("  children table", nodes["children"][:min(k, 8)])
ex.close()
