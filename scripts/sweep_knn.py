"""K1a tuning sweep at BASELINE cfg 2 sizes: per-kernel times (library launch-event profiler) for several
points-per-cell settings given as SWEEP="ppc,...", each checked bit-for-bit against the first.
Not a bench value."""
import sys, os, hashlib
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from glio_b200 import api, synth

W, Q, M = int(os.environ.get("W", 20)), int(os.environ.get("Q", 100000)), int(os.environ.get("M", 1000000))
P = synth.window_problem(W=W, Q=Q, M=M)
dmap = torch.from_numpy(P["map_xyz"]).cuda(); dscans = [torch.from_numpy(s).cuda() for s in P["scans"]]
ref = None
for ppc in os.environ.get("SWEEP", "8,6,12").split(","):
    os.environ["GLIO_PTS_PER_CELL"] = ppc
    ctx = api.Context(0)
    ctx.set_map(dmap); ctx.window_set_scans(dscans)
    nm = ctx.window_associate(P["poses_init"])          # warm-up
    ctx.lib_profile(True)
    for _ in range(4):
        nm = ctx.window_associate(P["poses_init"])
    ctx.synchronize()
    prof = ctx.lib_profile_read(); ctx.lib_profile(False)
    h = hashlib.sha256()
    for s in (0, W // 2, W - 1):
        m = ctx.get_matches(s, int(nm[s]))
        for k in sorted(m):
            if isinstance(m[k], np.ndarray): h.update(np.ascontiguousarray(m[k]).tobytes())
    dig = h.hexdigest()[:16]
    if ref is None: ref = (dig, nm.copy())
    same = dig == ref[0] and np.array_equal(nm, ref[1])
    line = " ".join("%s=%.3f" % (k.replace("k_", ""), v[0] / v[1]) for k, v in prof.items() if k.startswith("k_knn") or k.startswith("k_plane") or k in ("k_transform_hist", "k_order_scatter"))
    knn = sum(v[0] / v[1] for k, v in prof.items() if k.startswith("k_knn"))
    print("ppc=%s knn_total=%.3f ms exact=%s | %s" % (ppc, knn, same, line), flush=True)
    ctx.close()
