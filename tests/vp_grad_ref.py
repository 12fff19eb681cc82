"""Extended-precision replay of tph's closed-track velocity profile (oracle/tph_velprofile.py: _solver_fb_closed,
_solver_fb_acc_profile, calc_ax_poss, conv_filt) with its gradient: the reference of the velocity-profile adjoint
(csrc/vel_profile_core.cuh, profile_adjoint_thread).  Written from the oracle, not from the kernel.  Test
infrastructure, not product code.

Two runs:

* decide() -- float64, the oracle's statements with a ggv scale and a top speed, recording every discrete decision: the
  fixed-point iteration count of the initial profile and the table segment of each of its lookups, the v_max clip of
  V0, and per step of both passes over the doubled lap a branch code in the layout of the kernel's tape
  (VP_BR_* in the low byte; for a taken step the ggv segment + 1 in bits 8..15 and the machine segment + 1 -- or, for
  a backward step whose correction won, the correction's ggv segment + 1 -- in bits 16..23).  Its vx is the oracle's.
* replay() -- np.longdouble on a scalar reverse tape (Var), the function the forward evaluates with those decisions
  frozen: the gradient of g_lap * T + g_vx . vx with respect to kappa and el, T = sum 2 e_i / (v_i + v_i+1) (the
  closed form of the step times, DESIGN.md section 3.12).  The codes may come from outside (the kernel's own), so that
  a test can replay the kernel's decision where the two break a tie differently.  With pin, a radicand 1 - q^p that
  the forward evaluated at the rounding level (q = 1 in exact arithmetic: a step starting on the lateral limit) is
  taken at the forward's value, and _conditioning() states what float64 cannot resolve there at dyn_model_exp != 1.

Table segments follow one convention: the right-hand segment at a knot, clamped (segment -1, slope 0) below the first
knot and from the last knot on.
"""
import math

import numpy as np

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, "the velocity-profile gradient reference needs an 80-bit or quad long double"

ACTIVE, TAKEN, LEAVE, VTMP, CLAMP, MACH, CLAMP2 = 1, 2, 4, 8, 16, 32, 64
LOW = 0xff


# ---- the reverse tape --------------------------------------------------------------------------------------------------
class Var:
    """A long-double scalar on the tape: its value and (parent, d value / d parent) pairs.  Nodes are appended to the
    tape as they are made, so the reverse of the tape is a topological order."""
    __slots__ = ("v", "par", "g")
    tape = None

    def __init__(self, v, par=()):
        self.v, self.par, self.g = v, par, LD(0)
        if Var.tape is not None:
            Var.tape.append(self)

    def __add__(self, o):
        if isinstance(o, Var):
            return Var(self.v + o.v, ((self, LD(1)), (o, LD(1))))
        return Var(self.v + o, ((self, LD(1)),))

    __radd__ = __add__

    def __sub__(self, o):
        if isinstance(o, Var):
            return Var(self.v - o.v, ((self, LD(1)), (o, LD(-1))))
        return Var(self.v - o, ((self, LD(1)),))

    def __rsub__(self, o):
        return Var(o - self.v, ((self, LD(-1)),))

    def __neg__(self):
        return Var(-self.v, ((self, LD(-1)),))

    def __mul__(self, o):
        if isinstance(o, Var):
            return Var(self.v * o.v, ((self, o.v), (o, self.v)))
        return Var(self.v * o, ((self, LD(o)),))

    __rmul__ = __mul__

    def __truediv__(self, o):
        if isinstance(o, Var):
            q = self.v / o.v
            return Var(q, ((self, 1 / o.v), (o, -q / o.v)))
        return Var(self.v / o, ((self, 1 / LD(o)),))

    def __rtruediv__(self, o):
        q = o / self.v
        return Var(q, ((self, -q / self.v),))

    def __pow__(self, c):                       # constant exponent
        c = LD(c)
        y = self.v ** c
        return Var(y, ((self, c * self.v ** (c - 1) if self.v != 0 else LD(0)),))


def val(x):
    return x.v if isinstance(x, Var) else LD(x)


def vsqrt(x):
    if not isinstance(x, Var):
        return np.sqrt(LD(x))
    y = np.sqrt(x.v)
    return Var(y, ((x, 1 / (2 * y)),))


def backprop(out, tape):
    out.g = LD(1)
    for node in reversed(tape):
        g = node.g
        if g != 0:
            for p, d in node.par:
                p.g += g * d


# ---- tables ------------------------------------------------------------------------------------------------------------
def segment(x, xp):
    """The segment of xp the derivative of numpy.interp takes at x: the right-hand one at a knot, -1 outside
    [xp[0], xp[-1]) and for NaN."""
    if not (x >= xp[0]) or x >= xp[-1]:
        return -1
    return int(np.searchsorted(xp, x, side="right")) - 1


def interp_frozen(x, xp, fp, seg):
    """numpy.interp on segment seg (linear there), or the end value it clamps to."""
    if seg < 0:
        end = fp[0] if val(x) < (xp[0] + xp[-1]) / 2 else fp[-1]
        return LD(end)
    x0, x1, f0, f1 = (LD(v) for v in (xp[seg], xp[seg + 1], fp[seg], fp[seg + 1]))
    return (x - x0) * ((f1 - f0) / (x1 - x0)) + f0


def _setup(ggv, mach, scale):
    g = np.array(ggv, dtype=float)
    g[:, 1:] *= scale                           # the oracle's ggv_mod (the kernel's mul(fp, s) rounds alike)
    return g, np.array(mach, dtype=float)


# ---- the decision run (float64) ----------------------------------------------------------------------------------------
def _ax_poss(vx, radius, ggv, mach, p, cd, m, forward):
    """calc_ax_poss (no mu) and the code of its decisions: CLAMP, MACH, ggv segment + 1 << 8, machine segment + 1 << 16
    (forward only); and the radicand."""
    ax_max_tires = np.interp(vx, ggv[:, 0], ggv[:, 1])
    ay_max_tires = np.interp(vx, ggv[:, 0], ggv[:, 2])
    ay_used = math.pow(vx, 2) / radius
    radicand = 1.0 - math.pow(ay_used / ay_max_tires, p)
    code = (segment(vx, ggv[:, 0]) + 1) << 8
    if radicand > 0.0:
        ax_avail = ax_max_tires * math.pow(radicand, 1.0 / p)
    else:
        ax_avail = 0.0
        code |= CLAMP
    if forward:
        ax_mach = np.interp(vx, mach[:, 0], mach[:, 1])
        code |= (segment(vx, mach[:, 0]) + 1) << 16
        if ax_mach < ax_avail:                  # min(ax_avail_tires, ax_max_machines_tmp)
            code |= MACH
        ax_avail = min(ax_avail, ax_mach)
    ax_drag = -math.pow(vx, 2) * cd / m
    return (ax_avail + ax_drag if forward else ax_avail - ax_drag), code, radicand


def _pass(ggv, mach, v_max, radii, el, vx_profile, p, cd, m, backwards, n_steps):
    """_solver_fb_acc_profile over the doubled lap; (profile, codes [n_steps], radicands {step: (r1, r2)})."""
    no_points = vx_profile.size
    if backwards:
        radii, el, vx_profile = np.flipud(radii), np.flipud(el), np.flipud(vx_profile)
    vx_profile = np.copy(vx_profile)
    acc_inds = np.where(np.diff(vx_profile) > 0.0)[0]
    acc_inds_rel = list(acc_inds[np.insert(np.diff(acc_inds), 0, 2) > 1]) if acc_inds.size else []
    codes = np.zeros(2 * (no_points // 2), dtype=np.int64)
    rads = {}
    while acc_inds_rel:
        i = acc_inds_rel.pop(0)
        while i < no_points - 1:
            a, c1, r1 = _ax_poss(vx_profile[i], radii[i], ggv, mach, p, cd, m, not backwards)
            vpn = math.sqrt(math.pow(vx_profile[i], 2) + 2 * a * el[i])
            code, extra, r2 = ACTIVE, c1 & ~LOW | c1 & (CLAMP | MACH), None
            if backwards:
                a2, c2, r2 = _ax_poss(vpn, radii[i + 1], ggv, mach, p, cd, m, False)
                vtmp = math.sqrt(math.pow(vx_profile[i], 2) + 2 * a2 * el[i])
                if vtmp < vpn:
                    vpn = vtmp
                    code |= VTMP
                    extra |= (CLAMP2 if c2 & CLAMP else 0) | (c2 & 0xff00) << 8
            if vpn < vx_profile[i + 1]:
                vx_profile[i + 1] = vpn
                code |= TAKEN | extra               # the tape keeps a step's table decisions where it stored
                rads[i] = (r1, r2 if code & VTMP else None)
            if vpn > v_max:
                code |= LEAVE
            if i < n_steps:
                codes[i] = code
            i += 1
            if vpn > v_max or (acc_inds_rel and i >= acc_inds_rel[0]):
                break
    if backwards:
        vx_profile = np.flipud(vx_profile)
    return vx_profile, codes, rads


def decide(kappa, el, ggv, mach, v_max, scale=1.0, exp=1.0, filt=None, upper=True, drag_coeff=0.75, m_veh=1200.0):
    """The oracle's closed-track profile in float64 with its decisions.  Returns the log replay() takes:
    dict(vx [n] (the oracle's), codes [4n] (forward pass, then backward pass, as the kernel's tape), iters (index of
    the last fixed-point iteration), init_seg [iters + 1, n], V0 [n] (before the clip), clip [n], rads {(pass, j):
    (radicand of the step's ax_poss, of its correction or None)} for taken steps, and the problem)."""
    kappa, el = np.asarray(kappa, dtype=float), np.asarray(el, dtype=float)
    g, mc = _setup(ggv, mach, scale)
    n = kappa.size
    radii = np.abs(np.divide(1.0, kappa, out=np.full(n, np.inf), where=kappa != 0.0))
    ay_max_global = np.mean(np.ones(n)) * np.amin(g[:, 2])
    init_seg = []
    with np.errstate(invalid="ignore", divide="ignore"):
        vx = np.sqrt(ay_max_global * radii)
        for it in range(100):
            prev = vx
            init_seg.append([segment(v, g[:, 0]) for v in prev])
            vx = np.sqrt(np.multiply(np.ones(n) * np.interp(vx, g[:, 0], g[:, 2]), radii))
            if np.max(np.abs(vx / prev - 1.0)) < 0.005:
                break
    V0 = vx.copy()
    clip = V0 > v_max
    vx[clip] = v_max
    r2, e2 = np.concatenate((radii, radii)), np.concatenate((el, el))
    cd, m = drag_coeff, m_veh
    fwd, kf, rf = _pass(g, mc, v_max, r2, e2, np.concatenate((vx, vx)), exp, cd, m, False, 2 * n - 1)
    fwd = np.concatenate((fwd[n:], fwd[n:]))
    j_end = n - 1 if upper else 2 * n - 1          # the kernel stops where the kept half is complete
    bwd, kb, rb = _pass(g, mc, v_max, r2, e2, fwd, exp, cd, m, True, j_end)
    vx = bwd[n:] if upper else bwd[:n]
    if filt is not None and filt > 1:
        h = (filt - 1) // 2
        vx = np.convolve(np.concatenate((vx[-h:], vx, vx[:h])), np.ones(filt) / float(filt), mode="same")[h:-h]
    codes = np.concatenate((kf, kb)).astype(np.int32)
    rads = {**{("fwd", j): r for j, r in rf.items()}, **{("bwd", j): r for j, r in rb.items() if j < j_end}}
    return dict(vx=vx, codes=codes, iters=len(init_seg) - 1, init_seg=np.array(init_seg), V0=V0, clip=clip, rads=rads,
                ggv=g, mach=mc, v_max=float(v_max), exp=float(exp), filt=filt, upper=bool(upper), cd=cd, m=m)


# ---- the replay (long double, reverse tape) ----------------------------------------------------------------------------
def _ax_poss_frozen(v, radius, code, lg, forward, pin=None):
    """The frozen calc_ax_poss at v; pin: the radicand's value to use in place of the one evaluated here (its
    derivative is kept)."""
    g, p = lg["ggv"], lg["exp"]
    seg = ((code >> 8) & 0xff) - 1
    ax_t = interp_frozen(v, g[:, 0], g[:, 1], seg)
    ay_t = interp_frozen(v, g[:, 0], g[:, 2], seg)
    q = v * v / radius / ay_t
    rad = 1 - q if p == 1.0 else 1 - q ** p
    if pin is not None:
        rad = Var(LD(pin), rad.par) if isinstance(rad, Var) else LD(pin)
    if code & CLAMP:
        avail = LD(0)
    else:
        avail = ax_t * (rad if p == 1.0 else rad ** (1 / LD(p)))
    if forward:
        mc = lg["mach"]
        mach = interp_frozen(v, mc[:, 0], mc[:, 1], ((code >> 16) & 0xff) - 1)
        if code & MACH:
            avail = mach
    drag = v * v * LD(lg["cd"]) / LD(lg["m"])
    return (avail - drag if forward else avail + drag), (rad, val(q))


def replay(kappa, el, lg, g_lap=1.0, g_vx=None, codes=None, iters=None, tape=True, pin=None):
    """The frozen function of the log lg at (kappa, el) in long double.  codes / iters: decisions from outside in place
    of the log's (the init segments and the clip stay the log's; iters must then equal the log's).  Returns
    dict(vx [n], laptime, loss, g_kappa [n], g_el [n] (tape=True), rads {(pass, j): (radicand, radicand of the
    correction or None)})."""
    n = len(kappa)
    codes = lg["codes"] if codes is None else np.asarray(codes)
    if iters is not None and iters != lg["iters"]:
        raise ValueError("replay: the initial profile's iteration count differs from the log's")
    Var.tape = nodes = [] if tape else None
    try:
        K = [Var(LD(k)) for k in kappa]
        E = [Var(LD(e)) for e in el]
        R = [(1 / K[i] if kappa[i] > 0 else -1 / K[i]) if kappa[i] != 0 else LD(np.inf) for i in range(n)]
        g = lg["ggv"]
        ay_global = LD(np.amin(g[:, 2]))
        V0 = []
        for i in range(n):
            if lg["clip"][i]:
                V0.append(LD(lg["v_max"]))
                continue
            vp = vsqrt(ay_global * R[i])
            for it in range(lg["iters"] + 1):
                ay = interp_frozen(vp, g[:, 0], g[:, 2], int(lg["init_seg"][it, i]))
                vp = vsqrt(ay * R[i])
            V0.append(vp)
        calls = []                      # (step, call, point, clamped, radicand node, q) of every ax_poss a taken step ran

        def pinned(key, k):
            r = lg["rads"].get(key)
            return r[k] if pin is not None and r is not None and r[k] is not None and 0.0 < r[k] < pin else None

        # forward pass over the doubled lap; the second lap is kept
        vd = V0 + V0
        for j in range(2 * n - 1):
            c = int(codes[j])
            if c & ACTIVE and c & TAKEN:
                i0 = j % n
                a, r1 = _ax_poss_frozen(vd[j], R[i0], c, lg, True, pinned(("fwd", j), 0))
                calls.append((("fwd", j), 0, i0, c & CLAMP) + r1)
                vd[j + 1] = vsqrt(vd[j] * vd[j] + 2 * a * E[i0])

        # backward pass on the flipped doubled lap (vd[n:], vd[n:]); step j goes from original point 2n-1-j to 2n-2-j
        fl = (vd[n:] + vd[n:])[::-1]
        j_end = n - 1 if lg["upper"] else 2 * n - 1
        for j in range(j_end):
            c = int(codes[2 * n + j])
            if c & ACTIVE and c & TAKEN:
                i0, i1 = (2 * n - 1 - j) % n, (2 * n - 2 - j) % n
                cur = fl[j]
                a, r1 = _ax_poss_frozen(cur, R[i0], c, lg, False, pinned(("bwd", j), 0))
                calls.append((("bwd", j), 0, i0, c & CLAMP) + r1)
                vpn = vsqrt(cur * cur + 2 * a * E[i0])
                if c & VTMP:
                    c2 = ((c >> 16) & 0xff) << 8 | (CLAMP if c & CLAMP2 else 0)
                    a2, r2 = _ax_poss_frozen(vpn, R[i1], c2, lg, False, pinned(("bwd", j), 1))
                    calls.append((("bwd", j), 1, i1, c & CLAMP2) + r2)
                    vpn = vsqrt(cur * cur + 2 * a2 * E[i0])
                fl[j + 1] = vpn
        orig = fl[::-1]
        V = orig[n:] if lg["upper"] else orig[:n]
        f = lg["filt"]
        if f is not None and f > 1:
            h, w = (f - 1) // 2, LD(1.0 / float(f))
            V = [sum((V[(i + k) % n] * w for k in range(-h, h + 1)), LD(0)) for i in range(n)]
        T = sum((2 * E[i] / (V[i] + V[(i + 1) % n]) for i in range(n)), LD(0))
        loss = T * LD(g_lap)
        if g_vx is not None:
            loss = loss + sum((V[i] * LD(g_vx[i]) for i in range(n) if g_vx[i] != 0), LD(0))
        rads = {}
        for key, k, _, _, rad, _ in calls:
            rads.setdefault(key, [None, None])[k] = val(rad)
        out = dict(vx=np.array([val(v) for v in V], dtype=LD), laptime=val(T), loss=val(loss),
                   rads={key: tuple(r) for key, r in rads.items()})
        if tape and isinstance(loss, Var):
            backprop(loss, nodes)
            out["g_kappa"] = np.array([k.g for k in K], dtype=LD)
            out["g_el"] = np.array([e.g for e in E], dtype=LD)
        elif tape:
            out["g_kappa"], out["g_el"] = np.zeros(n, dtype=LD), np.zeros(n, dtype=LD)
        if tape:
            out["cond_kappa"] = _conditioning(calls, kappa, lg, pinned)
        return out
    finally:
        Var.tape = None


def _conditioning(calls, kappa, lg, pinned):
    """What float64 cannot resolve in dL/dkappa at dyn_model_exp p != 1, per point (0 at p = 1).

    A step's ax_poss evaluates rho = 1 - q^p with q = v^2 / (r ay_max) and uses rho^(1/p).  Its derivatives with respect
    to the carried speed and the radius are each of size A = |dL/drho| p q^p / |kappa| and, where the speed is the
    initial profile's lateral-limit speed of the same point (dq = 0 along it), they cancel: float64 keeps an absolute
    error of about u A of the sum.  And rho itself is a difference of numbers near 1, known to about u absolutely,
    so the factor rho^(1/p - 1) of both derivatives is known to about u / rho relatively (not where rho is pinned:
    there the reference uses the forward's own rho).  Returns, per point, the sum over its unclamped calls of
    u A (1 + 1 / rho), u = 2^-53."""
    u = 2.0 ** -53
    p = lg["exp"]
    cond = np.zeros(len(kappa))
    if p == 1.0:
        return cond
    for key, k, i, clamped, rad, q in calls:
        if clamped or not isinstance(rad, Var) or kappa[i] == 0.0:
            continue
        A = float(abs(rad.g)) * p * float(q) ** p / abs(kappa[i])
        r = lg["rads"].get(key)
        rho = r[k] if r is not None and r[k] is not None else float(rad.v)
        cond[i] += u * A * (1.0 + (0.0 if pinned(key, k) is not None else 1.0 / rho))
    return cond


def code_diffs(ref, kern, n, upper):
    """The steps whose codes differ: [(pass, j, ref code, kernel code)] (backward steps beyond the kept half are not
    run by the kernel)."""
    ref, kern = np.asarray(ref), np.asarray(kern)
    out = [("fwd", j, int(ref[j]), int(kern[j])) for j in range(2 * n - 1) if ref[j] != kern[j]]
    j_end = n - 1 if upper else 2 * n - 1
    out += [("bwd", j, int(ref[2 * n + j]), int(kern[2 * n + j])) for j in range(j_end)
            if ref[2 * n + j] != kern[2 * n + j]]
    return out
