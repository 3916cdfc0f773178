"""float32 numpy twin of the sphere-tracing state machine of csrc/surface.cu (BaseNeuralField.trace_surface).

Every float operation is one numpy float32 operation (each rounded to nearest, no fused multiply-add), in the order the
kernels perform them, so the twin matches the kernels bit for bit when it is fed the same field values.  ``field`` is a
callable ``(pos [m,3] float32, dir [m,3] float32) -> values [m] float32``; it sees the live rays of one pass in ray
order (the kernels' order varies; no result depends on it).

Besides the kernels' outputs the twin records, per ray, a decision-margin witness: the smallest of |g - EPS|, |g| and
|t_next - far| it met, i.e. how far the ray's trajectory was from taking another branch.
"""
import numpy as np

MARCH, BISECT, HIT, MISS = 0, 1, 16, 17
EPS = np.float32(1e-4)
FD_H = np.float32(1e-4)
BISECTIONS = 8
f32 = np.float32


def points(o, d, t):
    """o + t d per component: a rounded product, then a rounded sum."""
    return (o + (t[:, None] * d).astype(f32)).astype(f32)


def trace(field, ray_dir, ray_orig, near, far, level, max_steps, history=None):
    """-> dict t, state, steps (per ray), lo, hi, live_counts (after each pass), margin (float64 witness).
    ``history``, when a list, receives (live ray ids, values) of every pass."""
    d = np.ascontiguousarray(ray_dir, f32)
    o = np.ascontiguousarray(ray_orig, f32)
    n = d.shape[0]
    near, far, level = f32(near), f32(far), f32(level)
    t = np.full(n, near, f32)
    lo, hi = t.copy(), t.copy()
    state = np.full(n, MARCH, np.int32)
    steps = np.zeros(n, np.int32)
    margin = np.full(n, np.inf)
    counts = []
    live = np.arange(n)
    while live.size:
        v = np.asarray(field(points(o[live], d[live], t[live]), d[live]), f32).reshape(-1)
        if history is not None:
            history.append((live.copy(), v.copy()))
        g = (v - level).astype(f32)
        margin[live] = np.minimum(margin[live], np.minimum(np.abs(g.astype(np.float64) - float(EPS)),
                                                           np.abs(g.astype(np.float64))))
        tl, ll, hl, sl = t[live], lo[live], hi[live], state[live]
        used = steps[live] + 1
        march = sl == MARCH
        # MARCH
        step = march & (g >= EPS)
        tn = (tl + g).astype(f32)
        margin[live[step]] = np.minimum(margin[live[step]], np.abs(tn[step].astype(np.float64) - float(far)))
        ll = np.where(step, tl, ll)
        tl = np.where(step, tn, tl)
        sl = np.where(step & (tn > far), MISS, sl)
        sl = np.where(march & ~step & (g >= 0), HIT, sl)
        inside = march & (g < 0)
        sl = np.where(inside & (used == 1), MISS, sl)
        over = inside & (used > 1)
        hl = np.where(over, tl, hl)
        sl = np.where(over, BISECT, sl)
        # BISECT
        bis = ~march
        ll = np.where(bis & (g >= 0), tl, ll)
        hl = np.where(bis & (g < 0), tl, hl)
        sl = np.where(bis, sl + 1, sl)
        done = bis & (sl == BISECT + BISECTIONS)
        tl = np.where(done, ll, tl)
        sl = np.where(done, HIT, sl)
        mid = (sl >= BISECT) & (sl < BISECT + BISECTIONS)
        tmid = (ll + ((hl - ll).astype(f32) * f32(0.5)).astype(f32)).astype(f32)
        tl = np.where(mid, tmid, tl)
        sl = np.where((sl != HIT) & (sl != MISS) & (used >= max_steps), MISS, sl)
        tl = np.where(sl == MISS, far, tl).astype(f32)
        t[live], lo[live], hi[live], state[live], steps[live] = tl, ll, hl, sl.astype(np.int32), used
        live = live[(sl != HIT) & (sl != MISS)]
        counts.append(int(live.size))
    return {"t": t, "lo": lo, "hi": hi, "state": state, "steps": steps, "live_counts": counts, "margin": margin}


def fd_coord(x, sign):
    return (x + FD_H).astype(f32) if sign > 0 else (x - FD_H).astype(f32)


def fd_points(hit_pos, hit_dir):
    """6 points per hit (x+h, x-h, y+h, y-h, z+h, z-h) with the hit's direction: ([6m,3], [6m,3])."""
    p = np.ascontiguousarray(hit_pos, f32)
    pts = np.repeat(p, 6, axis=0).reshape(-1, 6, 3)
    for q in range(6):
        pts[:, q, q // 2] = fd_coord(p[:, q // 2], +1 if q % 2 == 0 else -1)
    return pts.reshape(-1, 3), np.repeat(np.ascontiguousarray(hit_dir, f32), 6, axis=0)


def fd_normals(values, hit_pos):
    """Unit normals [m,3] from the field at fd_points: differences over the rounded spacings, normalised."""
    v = np.asarray(values, f32).reshape(-1, 6)
    p = np.ascontiguousarray(hit_pos, f32)
    g = np.empty_like(p)
    for c in range(3):
        span = (fd_coord(p[:, c], +1) - fd_coord(p[:, c], -1)).astype(f32)
        g[:, c] = ((v[:, 2 * c] - v[:, 2 * c + 1]).astype(f32) / span).astype(f32)
    sq = (g * g).astype(f32)
    length = np.sqrt(((sq[:, 0] + sq[:, 1]).astype(f32) + sq[:, 2]).astype(f32)).astype(f32)
    safe = np.where(length > 0, length, f32(1))
    return np.where(length[:, None] > 0, (g / safe[:, None]).astype(f32), f32(0)).astype(f32)


# ---------------------------------------------------------------------------------------------- analytic fields --
def sphere_sdf(center, radius, scale=1.0):
    """scale * (|p - c| - r), every step rounded to fp32 (scale 2 overshoots and exercises the bisection)."""
    c, r, s = np.asarray(center, f32), f32(radius), f32(scale)

    def f(p, d):
        q = (p - c).astype(f32)
        sq = (q * q).astype(f32)
        dist = (np.sqrt(((sq[:, 0] + sq[:, 1]).astype(f32) + sq[:, 2]).astype(f32)).astype(f32) - r).astype(f32)
        return dist if s == 1 else (s * dist).astype(f32)
    return f


def plane_sdf(normal, offset):
    """n . p - offset for a unit n, rounded per operation."""
    nn_ = np.asarray(normal, f32)

    def f(p, d):
        pr = (p * nn_).astype(f32)
        return (((pr[:, 0] + pr[:, 1]).astype(f32) + pr[:, 2]).astype(f32) - f32(offset)).astype(f32)
    return f
