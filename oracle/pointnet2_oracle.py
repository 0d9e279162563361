"""numpy restatement of the pointnet2_ops operators as csrc/pn2_ops.cu computes them (include/gs_b200.h states the
rules).  Every float32 numpy operation rounds once, as the kernels do under -fmad=false, and each expression keeps the
kernels' operation order, so the results are bit-identical.  np.argmax's first-occurrence rule is the kernels'
smallest-index tie rule.  The backward folds are also given in float64 (dtype=np.float64) for gradient checks."""
import numpy as np

F32 = np.float32
ONCHIP_MAX = 16384           # GS_B200_PN2_FPS_ONCHIP_MAX: larger clouds take the global-memory FPS kernel


def _d2(a, b):
    """((dx*dx + dy*dy) + dz*dz) in the dtype of a and b; a and b broadcast against each other over [..., 3]."""
    d = a - b
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def fps_skipped(xyz):
    """pointnet2_ops' skip rule: fp32 (x*x + y*y) + z*z compared, as double, against 1e-3."""
    xyz = np.asarray(xyz, F32)
    mag = (xyz[..., 0] * xyz[..., 0] + xyz[..., 1] * xyz[..., 1]) + xyz[..., 2] * xyz[..., 2]
    return mag.astype(np.float64) <= 1e-3


def furthest_point_sample(xyz, npoint):
    """xyz [B,N,3] float32 -> int32 [B,npoint]."""
    xyz = np.asarray(xyz, F32)
    B, N, _ = xyz.shape
    out = np.zeros((B, npoint), np.int32)
    for b in range(B):
        p = xyz[b]
        temp = np.where(fps_skipped(p), F32(-1), F32(1e10)).astype(F32)
        last = 0
        for s in range(1, npoint):
            temp = np.fmin(_d2(p, p[last]), temp)          # fminf: a NaN distance leaves temp unchanged
            last = int(np.argmax(temp)) if temp.max() >= 0 else 0
            out[b, s] = last
    return out


def ball_query(radius, nsample, xyz, new_xyz):
    """xyz [B,N,3], new_xyz [B,P,3] float32 -> int32 [B,P,nsample]."""
    xyz, new_xyz = np.asarray(xyz, F32), np.asarray(new_xyz, F32)
    B, P = new_xyz.shape[:2]
    r2 = F32(radius) * F32(radius)
    out = np.zeros((B, P, nsample), np.int32)
    if nsample == 0:
        return out
    for b in range(B):
        hit = _d2(new_xyz[b][:, None, :], xyz[b][None, :, :]) < r2        # [P, N]
        for q in range(P):
            k = np.flatnonzero(hit[q])[:nsample]
            if k.size:
                out[b, q, :] = k[0]
                out[b, q, :k.size] = k
    return out


def three_nn(unknown, known):
    """unknown [B,n,3], known [B,m,3] float32 -> (dist float32 [B,n,3], idx int32 [B,n,3])."""
    unknown, known = np.asarray(unknown, F32), np.asarray(known, F32)
    B, n = unknown.shape[:2]
    dist = np.full((B, n, 3), np.inf, F32)
    idx = np.zeros((B, n, 3), np.int32)
    for b in range(B):
        d2 = _d2(unknown[b][:, None, :], known[b][None, :, :])             # [n, m]
        order = np.argsort(d2, axis=1, kind="stable")[:, :3]                # ascending d2, ascending k on ties; NaN last
        v = np.take_along_axis(d2, order, axis=1)
        ok = v < np.inf                                                     # NaN and +inf never enter
        k = order.shape[1]
        dist[b, :, :k] = np.where(ok, np.sqrt(v), F32(np.inf))
        idx[b, :, :k] = np.where(ok, order, 0)
    return dist, idx


def gather(features, idx):
    """features [B,C,N], idx [B,...] int -> [B,C,...]; 0 where idx lies outside [0,N)."""
    features, idx = np.asarray(features), np.asarray(idx)
    B, C, N = features.shape
    ok = (idx >= 0) & (idx < N)
    safe = np.where(ok, idx, 0).reshape(B, 1, -1)
    out = np.take_along_axis(features, np.broadcast_to(safe, (B, C, safe.shape[2])), axis=2)
    out = np.where(ok.reshape(B, 1, -1), out, features.dtype.type(0))
    return out.reshape((B, C) + idx.shape[1:])


def three_interpolate(features, idx, weight):
    """features [B,C,m], idx [B,n,3], weight [B,n,3] -> (w0*f0 + w1*f1) + w2*f2, f = 0 outside [0,m)."""
    features, weight = np.asarray(features), np.asarray(weight)
    f = gather(features, idx)                                               # [B,C,n,3]
    w = weight[:, None, :, :]
    return (w[..., 0] * f[..., 0] + w[..., 1] * f[..., 1]) + w[..., 2] * f[..., 2]


def _fold(vals, idx, N, dtype):
    """grad [B,C,N]: +0 plus vals [B,C,M] through idx [B,M], in ascending position, one add each; idx outside
    [0,N) skipped."""
    vals = np.asarray(vals, dtype)
    B, C, M = vals.shape
    idx = np.asarray(idx).reshape(B, M)
    out = np.zeros((B, C, N), dtype)
    for b in range(B):
        ok = (idx[b] >= 0) & (idx[b] < N)
        np.add.at(out[b].T, idx[b][ok], vals[b][:, ok].T)              # sequential in ascending position
    return out


def gather_grad(grad_out, idx, N, dtype=F32):
    """Backward of gather / grouping: grad_out [B,C,...] with idx [B,...]."""
    g = np.asarray(grad_out, dtype)
    return _fold(g.reshape(g.shape[0], g.shape[1], -1), idx, N, dtype)


def three_interpolate_grad(grad_out, idx, weight, m, dtype=F32):
    """Backward of three_interpolate for features: contributions grad_out[b,c,i] * weight[b,i,k] (rounded once) at
    position 3i + k."""
    g = np.asarray(grad_out, dtype)
    w = np.asarray(weight, dtype)
    B, C, n = g.shape
    vals = (g[:, :, :, None] * w[:, None, :, :]).reshape(B, C, n * 3)
    return _fold(vals, np.asarray(idx).reshape(B, n * 3), m, dtype)


def golden_calls(path):
    """The calls recorded in tests/golden/ref_pointnet2.npz (make_golden_pointnet2.py), as a list of dicts; an argument
    stored once and repeated is resolved."""
    z = np.load(path)
    calls = []
    for i in range(int(z["n_calls"])):
        pre = f"c{i}_"
        r = {}
        for k in z.files:
            if k.startswith(pre):
                v = z[k]
                if v.dtype.kind == "U" and str(v).startswith("@"):
                    v = z[str(v)[1:]]
                r[k[len(pre):]] = v
        r["op"], r["site"] = str(r["op"]), str(r["site"])
        calls.append(r)
    return calls


def replay(call):
    """The oracle's results for one recorded call: {name: array} for out (or dist and idx) and grad_features."""
    op = call["op"]
    if op == "furthest_point_sample":
        return {"out": furthest_point_sample(call["xyz"], int(call["npoint"]))}
    if op == "ball_query":
        return {"out": ball_query(float(call["radius"]), int(call["nsample"]), call["xyz"], call["new_xyz"])}
    if op == "three_nn":
        d, i = three_nn(call["unknown"], call["known"])
        return {"dist": d, "idx": i}
    res = {}
    if op in ("gather_operation", "grouping_operation"):
        res["out"] = gather(call["features"], call["idx"])
        if "grad_out" in call:
            res["grad_features"] = gather_grad(call["grad_out"], call["idx"], call["features"].shape[2])
    else:
        res["out"] = three_interpolate(call["features"], call["idx"], call["weight"])
        if "grad_out" in call:
            res["grad_features"] = three_interpolate_grad(call["grad_out"], call["idx"], call["weight"],
                                                          call["features"].shape[2])
    return res
