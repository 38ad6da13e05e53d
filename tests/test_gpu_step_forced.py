"""The env-step kernel one forced step at a time against the CPU oracle (oracle/env.h).

Free-running comparisons (test_gpu_parity.py, test_gpu_scenarios.py) cannot be tight: contacts amplify rounding over hundreds of
steps.  Here every env-step starts from the oracle's own state: its (q, qd, held torque, contact bits) are copied into each GPU
env, both sides take one env-step (physics sub-steps, decision, controller), and what is left is one step's disagreement.  The
controller blocks are not copied; they follow from the forced states and must stay in agreement on their own.

Per env and step: q, qd, held torque, every double of the controller block, and on decision steps the policy state and the net
output, as max|g - o| / (1 + |o|) <= 1e-10.  Contact bits, gait state, stance, action id and the integer fields of the
controller block are compared exactly.  Some stress states are stiff: there a second oracle steps from the state perturbed by
1e-15 relative, and q, qd and the held torque are held to 100x that sensitivity where it exceeds 1e-10 (Sensitivity), but never
to more than 1e-8, and at most 1 % of the comparisons may need it; the report lists those bounds.  The per-step worst on an H100
80GB HBM3 (700 W) is 3.7e-11 (qd); 8 of about 32,000 vertex-contact comparisons needed the wider bound, the largest error there
3.8e-9 in qd (dog), where 100x the oracle's sensitivity is 4.6e-7.

Stress states push the step into the branches ordinary gait rarely reaches: joints past their limits, clamped torques, deep and
near contacts, both friction regimes, corners inside the broad phase's margin, bodies over the seam between the two ground
segments, and the opt-in vertex contact model.  Each kind asserts, on the oracle side, that its branch was reached.

The helpers also drive tests/test_simt_cpu.py::test_forced_steps_and_stress_states_vs_oracle on the emulator."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

H = 1.0 / 600.0
TOL = 1e-10
CONTACT_TOL = 0.00025          # PhysParams.contact_tol (oracle/env.h, csrc/trl_types.h)
V_EPS = 0.01                   # PhysParams.v_eps
CLEAR_MARGIN = 0.05            # kClearMargin (csrc/trl_step.cu)
SPACING = 0.1                  # terrain vertex spacing
FLOOR_CAP = 1e-8               # a stiff state's bound never exceeds this
STIFF_SHARE = 0.01             # at most this share of the comparisons may need more than the plain bound
KINDS = ("limit", "clamp", "deep", "near", "friction", "broad", "seam")


def _relerr(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.max(np.abs(a - b) / (1.0 + np.abs(b)))) if a.size else 0.0


# --------------------------------------------------------------------------------------------------- the character's geometry
class Model:
    """The pack's joint / body tables (as oracle/rbd.h reads them) and the planar kinematics of oracle/env.h: update_kin."""

    def __init__(self, pack):
        from pack_scene import read_pack
        p = read_pack(pack)
        mi = p["meta_i32"]
        self.char_type, self.ns, self.has_net = int(mi[0]), int(mi[3]), int(mi[7])
        self.nj, self.ndof = int(mi[8]), int(mi[9])
        J, B = p["joints"].reshape(self.nj, 7), p["bodies"].reshape(self.nj, 9)
        self.parent = J[:, 1].astype(int)
        self.attach = J[:, 2:4]
        self.lo, self.hi = J[:, 5], J[:, 6]
        self.offset = np.array([0] + [2 + j for j in range(1, self.nj)])
        self.battach, self.btheta, self.half = B[:, 2:4], B[:, 5], 0.5 * B[:, 6:8]
        self.tmax = p["pd"].reshape(self.nj, 6)[:, 2]
        valid = B[:, 0] >= 0
        tail = np.zeros(self.nj, bool)
        if self.char_type == 1:
            tail[9:13] = True          # the dog's and goat's tail parts do not collide
        self.collide = valid & ~tail
        self.limited = [j for j in range(1, self.nj) if self.lo[j] <= self.hi[j]]
        # csrc/trl_host.cu: reach = upper bound of |corner - root joint| over all poses
        jr = np.zeros(self.nj)
        self.reach = 0.0
        for j in range(1, self.nj):
            jr[j] = jr[self.parent[j]] + np.hypot(*self.attach[j])
        for j in np.flatnonzero(self.collide):
            c, s = np.cos(self.btheta[j]), np.sin(self.btheta[j])
            for cn in range(4):
                bx = self.half[j, 0] * (1 if cn & 1 else -1)
                by = self.half[j, 1] * (1 if cn & 2 else -1)
                lx, ly = self.battach[j, 0] + c * bx - s * by, self.battach[j, 1] + s * bx + c * by
                self.reach = max(self.reach, jr[j] + np.hypot(lx, ly))

    def bodies(self, q, qd):
        """per body: centre (px, py), angle, centre velocity (vx, vy), angular velocity"""
        n = self.nj
        jp, jv = np.zeros((n, 2)), np.zeros((n, 2))
        ja, jw = np.zeros(n), np.zeros(n)
        out = np.zeros((n, 6))
        for j in range(n):
            p = self.parent[j]
            if p < 0:
                jp[j], ja[j], jv[j], jw[j] = q[0:2], q[2], qd[0:2], qd[2]
            else:
                c, s = np.cos(ja[p]), np.sin(ja[p])
                ax, ay = c * self.attach[j, 0] - s * self.attach[j, 1], s * self.attach[j, 0] + c * self.attach[j, 1]
                jp[j] = jp[p] + (ax, ay)
                ja[j] = ja[p] + q[self.offset[j]]
                jv[j] = jv[p] + (-jw[p] * ay, jw[p] * ax)
                jw[j] = jw[p] + qd[self.offset[j]]
            c, s = np.cos(ja[j]), np.sin(ja[j])
            bx, by = c * self.battach[j, 0] - s * self.battach[j, 1], s * self.battach[j, 0] + c * self.battach[j, 1]
            out[j] = (jp[j, 0] + bx, jp[j, 1] + by, ja[j] + self.btheta[j], jv[j, 0] - jw[j] * by, jv[j, 1] + jw[j] * bx, jw[j])
        return out

    def corners(self, q, qd):
        """rows (body, corner, x, y, vx, vy) of every collidable box corner, in the oracle's corner order"""
        rows = []
        for j, (px, py, ang, vx, vy, w) in enumerate(self.bodies(q, qd)):
            if not self.collide[j]:
                continue
            c, s = np.cos(ang), np.sin(ang)
            for cn in range(4):
                lx = self.half[j, 0] * (1 if cn & 1 else -1)
                ly = self.half[j, 1] * (1 if cn & 2 else -1)
                rx, ry = c * lx - s * ly, s * lx + c * ly
                rows.append((j, cn, px + rx, py + ry, vx - w * ry, vy + w * rx))
        return np.array(rows)


class Ground:
    """One env's ground as the oracle holds it (two segments, oracle/terrain.h: Ground)."""

    def __init__(self, o, env):
        self.o, self.env = o, env
        segs = [o.terrain(env, s) for s in (0, 1)]
        flip = segs[0][2]
        self.segs = [segs[1], segs[0]] if flip else segs          # [min segment, max segment]
        d, mx, _ = self.segs[0]
        self.seam = mx + (d.size - 1) * SPACING

    def height(self, x):
        return self.o.sample_height(float(x), self.env)

    def slope(self, x):
        e = 1e-7
        return (self.height(x + e) - self.height(x - e)) / (2 * e)

    def pen(self, x, y):
        """penetration of the point along the surface normal and the normal's (inv) factor, as oracle/env.h: forward_dynamics"""
        s = self.slope(x)
        inv = 1.0 / np.sqrt(1.0 + s * s)
        return (self.height(x) - y) * inv, s, inv

    def window_max(self, x0, x1):
        """GroundView::window_max (csrc/trl_terrain.cuh): the terrain maximum the kernel's broad phase uses"""
        return self.window_max_at(x0, x1)[0]

    def window_max_at(self, x0, x1):
        """the window maximum and the x of a vertex that attains it"""
        mx, at = -np.inf, None
        for d, mnx, _ in self.segs:
            w = d.size
            if w == 0:
                continue
            c0 = min(max((x0 - mnx) / SPACING, 0.0), w - 1.0)
            c1 = min(max((x1 - mnx) / SPACING, 0.0), w - 1.0)
            i0, i1 = int(c0), min(w - 1, int(c1) + 1)
            k = i0 + int(np.argmax(d[i0:i1 + 1]))
            if float(d[k]) > mx:
                mx, at = float(d[k]), mnx + k * SPACING
        return mx, at

    def vertices(self, x0, x1):
        """(x, h, h_prev, h_next) of the terrain vertices in [x0, x1] in the order Ground::for_vertices visits them"""
        out = []
        for si, (d, mnx, _) in enumerate(self.segs):
            w = d.size
            k0 = max(int(np.ceil((x0 - mnx) / SPACING - 1e-9)), 0)
            k1 = min(int(np.floor((x1 - mnx) / SPACING + 1e-9)), w - 1)
            for k in range(k0, k1 + 1):
                x = mnx + k * SPACING
                if (si == 0 and x >= self.seam) or (si == 1 and x < self.seam):
                    continue
                hp = float(d[k - 1]) if k > 0 else (self.height(x - SPACING) if si == 1 else float(d[k]))
                hn = float(d[k + 1]) if k < w - 1 else (self.height(x + SPACING) if si == 0 else float(d[k]))
                out.append((x, float(d[k]), hp, hn))
        return out


def corner_pens(m, o, env, q, qd):
    """corners with their penetration, normal factor and tangential speed"""
    gr = Ground(o, env)
    rows = []
    for j, cn, x, y, vx, vy in m.corners(q, qd):
        pen, s, inv = gr.pen(x, y)
        rows.append((j, cn, x, y, pen, inv, vx * inv + vy * s * inv))
    return np.array(rows), gr


# --------------------------------------------------------------------------------------------------- the forcing harness
def make_pair(assets, scene, n, mode=0, seeds=None, rng_seed=1234):
    from pyoracle import Oracle
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, scene + ".trlpack")
    seeds = list(range(101, 101 + n)) if seeds is None else list(seeds)
    cls = trl.ScenarioExpMACE if mode else trl.ScenarioPoliEval
    g = cls(pack, n, terrain_seeds=seeds, rng_seed=rng_seed)
    o = Oracle(pack, n, mode, terrain_seeds=seeds, rng_seed=rng_seed)
    return g, o, Model(pack)


def int_fields(m_params, nj):
    """indices of the integer fields of the controller block (trl_get_ctrl / orc_get_ctrl): state, first_cycle, action id, and
    fail flag, exp flags, cycle count, stance at the end"""
    n = 12 + m_params + nj + 5 + 5
    return np.array([0, 2, 11, n - 5, n - 4, n - 3, n - 2, n - 1]), n


class Worst:
    """worst relative error per (scene, quantity); the failures are collected, so that one run reports every figure"""

    def __init__(self, tol=TOL):
        self.tol, self.w, self.fail = tol, {}, []     # tol: one bound, or {quantity: bound} with a "default"
        self.stiff, self.n, self.needed = {}, 0, 0

    def rel(self, key, what, g, o, where, floor=0.0):
        """floor: 100 x the oracle's own sensitivity at this state (see Sensitivity); a stiff state is held to that instead, but
        never to more than FLOOR_CAP, and report() fails if more than STIFF_SHARE of the comparisons needed the floor"""
        e = _relerr(g, o)
        k = (key, what)
        self.w[k] = max(self.w.get(k, 0.0), e)
        self.n += 1
        tol = self.tol.get(what, self.tol["default"]) if isinstance(self.tol, dict) else self.tol
        if floor > tol:
            self.stiff[k] = max(self.stiff.get(k, (0.0, 0.0)), (min(floor, FLOOR_CAP), e))
            if e > tol:
                self.needed += 1
            tol = min(floor, FLOOR_CAP)
        if not e <= tol:
            self.fail.append((key, what, where, e))

    def exact(self, key, what, g, o, where):
        if not np.array_equal(np.asarray(g), np.asarray(o)):
            self.fail.append((key, what, where, "differs: %s vs %s" % (np.asarray(g).tolist(), np.asarray(o).tolist())))

    def report(self):
        for (key, what), e in sorted(self.w.items()):
            print("forced %-34s %-11s worst %.2e" % (key, what, e))
        for (key, what), (b, e) in sorted(self.stiff.items()):
            print("stiff  %-34s %-11s largest bound %.2e (100 x sensitivity), error there %.2e" % (key, what, b, e))
        print("stiff  %d of %d comparisons passed only through the sensitivity bound" % (self.needed, self.n))
        assert not self.fail, self.fail[:12]
        assert self.needed <= STIFF_SHARE * self.n, (self.needed, self.n)


def force(g, o, envs):
    for e in envs:
        q, qd, tau, c = o.get_state(e)
        g.SetState(e, q=q, qd=qd, tau=tau, contact=c)


def compare(g, o, envs, worst, key, step, ints, net_out_n, sens=None):
    """one forced step's results for each env; returns the envs that took a decision in it"""
    decided = []
    for e in envs:
        where = (step, e)
        fl = sens.floor[e] if sens is not None else {}
        gq, gqd, gt, gc = g.GetState(e)
        oq, oqd, ot, oc = o.get_state(e)
        worst.rel(key, "q", gq, oq, where, fl.get("q", 0.0))
        worst.rel(key, "qd", gqd, oqd, where, fl.get("qd", 0.0))
        worst.rel(key, "tau", gt, ot, where, fl.get("tau", 0.0))
        worst.exact(key, "contact", gc, oc, where)
        gk, ok = g.GetCtrl(e), o.get_ctrl(e)
        if gk.size != ok.size:
            worst.fail.append((key, "ctrl size", where, (gk.size, ok.size)))
            continue
        dbl = np.ones(ok.size, bool)
        dbl[ints] = False
        worst.rel(key, "ctrl", gk[dbl], ok[dbl], where)
        worst.exact(key, "ctrl ints", gk[ints], ok[ints], where)
        if ok[0] == 0 and ok[1] == 0:              # state 0 at phase 0: the env took a decision in this step
            decided.append(e)
            worst.rel(key, "poli state", g.GetPoliState(e), o.poli_state(e), where)
            if net_out_n:
                worst.rel(key, "net out", g.GetNetOut(e, net_out_n), o.net_out(e, net_out_n), where)
    return decided


class Sensitivity:
    """A second oracle, forced like the GPU, that takes every step from the oracle's state perturbed by 1e-15 relative.  How far
    its q, qd and held torque land from the oracle's is the problem's own conditioning at that state: a GPU difference within
    100x of it is rounding amplified by a stiff state, not a kernel error."""

    def __init__(self, assets, scene, n, mode=0, seeds=None, rng_seed=1234):
        from pyoracle import Oracle
        seeds = list(range(101, 101 + n)) if seeds is None else list(seeds)
        self.o = Oracle(os.path.join(assets, scene + ".trlpack"), n, mode, terrain_seeds=seeds, rng_seed=rng_seed)
        self.rng = np.random.default_rng(0)
        self.floor = {}

    def install(self, o, envs):
        for e in envs:
            q, qd, tau, c = o.get_state(e)
            wig = lambda a: a * (1.0 + 1e-15 * self.rng.standard_normal(a.size))
            self.o.set_state(e, wig(q), wig(qd), tau, c)

    def step(self, o, envs):
        for e in envs:
            self.o.env_step(e, H)
            a, b = o.get_state(e), self.o.get_state(e)
            self.floor[e] = {"q": 100 * _relerr(b[0], a[0]), "qd": 100 * _relerr(b[1], a[1]), "tau": 100 * _relerr(b[2], a[2])}


def step_all(g, o, envs, shadow=None, sens=None):
    """force, then one env-step on both sides.  A shadow oracle (the other contact model) takes the step from the same states;
    returns whether its physics disagrees with the oracle's for some env"""
    force(g, o, envs)
    if shadow is not None:
        for e in envs:
            shadow.set_state(e, *o.get_state(e))
    if sens is not None:
        sens.install(o, envs)
    g.EnvStep(H)
    for e in envs:
        o.env_step(e, H)
    if sens is not None:
        sens.step(o, envs)
    if shadow is None:
        return False
    differ = False
    for e in envs:
        shadow.env_step(e, H)
        a, b = o.get_state(e), shadow.get_state(e)
        differ |= not all(np.array_equal(a[i], b[i]) for i in (0, 1, 3))
    return differ


def forced_steps(g, o, m, envs, steps, worst, key, shadow=None, stats=None, sens=None):
    ints, _ = int_fields(n_params(o), m.nj)
    nout = net_out_size(g, m)
    decisions = 0
    for k in range(steps):
        differ = step_all(g, o, envs, shadow, sens)
        if stats is not None:
            stats["model mattered"] = stats.get("model mattered", 0) + int(differ)
        decisions += len(compare(g, o, envs, worst, key, k, ints, nout, sens))
    return decisions


def n_params(o):
    return o.get_ctrl(0).size - 12 - o.nj - 10


def net_out_size(g, m):
    return g.num_frags * (1 + g.frag_size) if m.has_net else 0


# --------------------------------------------------------------------------------------------------- stress states
def lift_to(q, corner_pen, corner_inv, target):
    """raise the root so that a corner whose penetration is corner_pen gets target"""
    q = q.copy()
    q[1] += (corner_pen - target) / corner_inv
    return q


def stress_state(kind, variant, rng, m, o, env, q, qd, tau):
    """a perturbed copy of (q, qd, tau) that reaches `kind`'s branch; `variant` (how often the kind was drawn before) alternates
    between its two sides: friction below / above v_eps, near contact at pen <= 0 / pen > 0, broad phase near / far from the
    window maximum"""
    q, qd, tau = q.copy(), qd.copy(), tau.copy()
    q[0] += rng.uniform(-0.02, 0.02)
    if kind == "limit":
        for j in rng.choice(m.limited, size=2, replace=False):
            o_ = m.offset[j]
            if rng.uniform() < 0.5:
                q[o_], qd[o_] = m.hi[j] + rng.uniform(0.02, 0.3), rng.uniform(0.2, 3.0)
            else:
                q[o_], qd[o_] = m.lo[j] - rng.uniform(0.02, 0.3), -rng.uniform(0.2, 3.0)
        cp, _ = corner_pens(m, o, env, q, qd)
        i = np.argmax(cp[:, 4])
        return lift_to(q, cp[i, 4], cp[i, 5], rng.uniform(-0.01, 0.002)), qd, tau
    if kind == "clamp":
        qd[3:] *= rng.uniform(3.0, 10.0)
        return q, qd, tau
    cp, gr = corner_pens(m, o, env, q, qd)
    order = np.argsort(-cp[:, 4])
    if kind == "deep":
        i = order[1]                                  # the second deepest corner: two or more penetrate
        return lift_to(q, cp[i, 4], cp[i, 5], rng.uniform(0.001, 0.012)), qd, tau
    if kind == "near":
        # at rest and without torque, so that the corners stay inside the band over the sub-steps (gravity alone moves them
        # 0.014 mm in an env-step)
        qd[:] = 0.0
        tau[:] = 0.0
        i = order[0]
        pen = rng.uniform(-0.9, -0.3) if variant % 2 == 0 else rng.uniform(0.05, 0.9)
        return lift_to(q, cp[i, 4], cp[i, 5], pen * CONTACT_TOL), qd, tau
    if kind == "friction":
        # rigid translation only: every point moves at (vx, 0), so the tangential speeds are vx * inv on a slope of the feet
        qd[:] = 0.0
        qd[0] = rng.choice([-1, 1]) * (rng.uniform(0.001, 0.006) if variant % 2 == 0 else rng.uniform(0.03, 1.0))
        i = order[0]
        return lift_to(q, cp[i, 4], cp[i, 5], rng.uniform(0.0005, 0.004)), qd, tau
    if kind == "broad":
        # the lowest corner between the kernel's window maximum and that maximum + kClearMargin.  Every other draw it sits over the
        # vertex that attains the maximum, 0.03 .. 0.5 contact_tol above it: above the maximum, so only the margin keeps it a
        # candidate, and inside the touching band all the same.  The other draws put it 0.2 .. 45 mm above (a candidate that
        # touches nothing).  The root moves along x (by the least amount, at most 3 m) so that the corner lies over a vertex that
        # is the maximum of the window around the moved root.
        i = np.argmin(cp[:, 3])                       # translating the character keeps it the lowest corner
        if variant % 2 == 0:
            best = None
            for xv, hv, _, _ in gr.vertices(cp[i, 2] - 3.0, cp[i, 2] + 3.0):
                dx = xv - cp[i, 2]
                if gr.window_max(q[0] + dx - m.reach - 0.25, q[0] + dx + m.reach + 0.25) == hv and (best is None or abs(dx) < abs(best[0])):
                    best = (dx, xv)
            if best is not None:
                xv = best[1]
                slope_l = (gr.height(xv) - gr.height(xv - 1e-4)) / 1e-4
                slope_r = (gr.height(xv + 1e-4) - gr.height(xv)) / 1e-4
                q[0] += xv + (1e-6 if abs(slope_r) < abs(slope_l) else -1e-6) - cp[i, 2]
                cp, _ = corner_pens(m, o, env, q, qd)
            gap = rng.uniform(0.03, 0.5) * CONTACT_TOL
        else:
            gap = rng.uniform(2e-4, 0.9 * CLEAR_MARGIN)
        wm = gr.window_max(q[0] - m.reach - 0.25, q[0] + m.reach + 0.25)
        q[1] += wm + gap - cp[i, 3]
        return q, qd, tau
    if kind == "seam":
        # a low body's centre onto the seam, then its lowest corner 0.5 .. 3 mm into the ground
        b = int(cp[order[0], 0])
        bx = m.bodies(q, qd)[b, 0]
        q[0] += gr.seam + rng.uniform(-0.3, 0.3) * m.half[b, 0] - bx
        cp, _ = corner_pens(m, o, env, q, qd)
        mine = cp[cp[:, 0] == b]
        i = np.argmax(mine[:, 4])
        return lift_to(q, mine[i, 4], mine[i, 5], rng.uniform(0.0005, 0.003)), qd, tau
    if kind == "vertex":
        # a convex terrain vertex 1 .. 4 mm inside the box of the longest collidable body, near the box's leading end so that it is
        # the last of the up to 4 vertices under the box (slot 3); every other draw a convex vertex past the seam.  Of the
        # candidate vertices the one that leaves the box corners least deep in the ground is taken (a placement that buries
        # another body makes the state blow up within a few steps).
        convex = lambda vs: [v for v in vs if v[1] - 0.5 * (v[2] + v[3]) > 1e-6]
        cands = convex(gr.vertices(gr.seam, gr.seam + 2.0)) if variant % 2 == 1 else []
        cands = cands or convex(gr.vertices(q[0] - 1.5, q[0] + 1.5))
        if not cands:
            return q, qd, tau
        qd *= 0.2
        bod = m.bodies(q, qd)
        ext = lambda j, a: abs(np.cos(a)) * m.half[j, 0] + abs(np.sin(a)) * m.half[j, 1]
        b = max(np.flatnonzero(m.collide), key=lambda j: ext(j, bod[j, 2]))
        if 2 * ext(b, bod[b, 2]) < 3 * SPACING + 0.01:
            # no box spans 4 vertices in this pose (the raptor's largest, 0.256 x 0.229 m, does so only turned near 42 degrees):
            # turn the character so that the box with the longest diagonal has it level
            b = max(np.flatnonzero(m.collide), key=lambda j: np.hypot(*m.half[j]))
            th = np.arctan2(m.half[b, 1], m.half[b, 0])
            turn = [np.angle(np.exp(1j * (t - bod[b, 2]))) for t in (th, -th, np.pi - th, th - np.pi)]
            q[2] += min(turn, key=abs)
            bod = m.bodies(q, qd)
        c, s_ = np.cos(bod[b, 2]), np.sin(bod[b, 2])
        hx, hy = m.half[b]
        best = None
        for sx in (-1, 1):
            for sy in (-1, 1):
                lx, ly = sx * (hx - rng.uniform(0.002, 0.01)), sy * (hy - rng.uniform(0.001, 0.004))
                wx, wy = c * lx - s_ * ly, s_ * lx + c * ly
                if best is None or (wx, -wy) > (best[0], -best[1]):
                    best = (wx, wy)
        placed = []
        for v in cands:
            qv = q.copy()
            qv[0] += v[0] - (bod[b, 0] + best[0])
            qv[1] += v[1] - (bod[b, 1] + best[1])
            placed.append((corner_pens(m, o, env, qv, qd)[0][:, 4].max(), qv))
        return min(placed, key=lambda t: t[0])[1], qd, tau
    raise ValueError(kind)


class Coverage:
    """oracle-side evidence that each stress kind reached its branch"""

    def __init__(self):
        self.c = {k: 0 for k in ("past limit", "clamped", "deep corners", "touching, no force", "slow friction", "fast friction",
                                 "in margin", "over seam", "vertex slot 3", "vertex past seam", "model mattered", "resets")}

    def at_install(self, kind, m, o, env, q, qd):
        cp, gr = corner_pens(m, o, env, q, qd)
        if kind == "limit":
            self.c["past limit"] += sum(1 for j in m.limited if not m.lo[j] <= q[m.offset[j]] <= m.hi[j])
        elif kind == "deep":
            self.c["deep corners"] += int(np.sum((cp[:, 4] >= 0.001) & (cp[:, 4] <= 0.02)) >= 2)
        elif kind == "friction":
            touching = cp[:, 4] > 0
            self.c["slow friction"] += int(np.sum(touching & (np.abs(cp[:, 6]) < V_EPS)))
            self.c["fast friction"] += int(np.sum(touching & (np.abs(cp[:, 6]) > V_EPS)))
        elif kind == "broad":
            # corners above the window maximum, so candidates only through kClearMargin, yet inside the touching band
            wm = gr.window_max(q[0] - m.reach - 0.25, q[0] + m.reach + 0.25)
            self.c["in margin"] += int(np.sum((cp[:, 3] > wm) & (cp[:, 3] <= wm + CLEAR_MARGIN) & (cp[:, 4] > -CONTACT_TOL)))
        elif kind == "seam":
            for b in np.unique(cp[:, 0]):
                xs = cp[cp[:, 0] == b, 2]
                self.c["over seam"] += int(xs.min() < gr.seam < xs.max())
        return cp

    def vertices_at_install(self, m, o, env, q):
        """the vertex contact model (oracle/env.h: forward_dynamics, GroundView::vertex_slot): for every body, the convex terrain
        vertices inside its box, by their slot in the body's window (the kernel looks at slots 0 .. 3)"""
        gr = Ground(o, env)
        for j, (px, py, ang, _, _, _) in enumerate(m.bodies(q, np.zeros_like(q))):
            if not m.collide[j]:
                continue
            c, s = np.cos(ang), np.sin(ang)
            hx, hy = m.half[j]
            ext = abs(c) * hx + abs(s) * hy
            vs = gr.vertices(px - ext - CONTACT_TOL, px + ext + CONTACT_TOL)
            assert len(vs) <= 4, (j, len(vs))
            for slot, (x, h, hp, hn) in enumerate(vs):
                if not h - 0.5 * (hp + hn) > 1e-9:
                    continue
                rx, ry = x - px, h - py
                lx, ly = c * rx + s * ry, -s * rx + c * ry
                if hx - abs(lx) > -CONTACT_TOL and hy - abs(ly) > -CONTACT_TOL:
                    self.c["vertex slot 3"] += int(slot == 3)
                    self.c["vertex past seam"] += int(x >= gr.seam > px - ext - CONTACT_TOL)

    def after_step(self, kind, m, o, env, cp_before):
        q, qd, _, c = o.get_state(env)
        if kind == "clamp":
            t = o.last_tau(env)
            self.c["clamped"] += sum(1 for j in range(1, m.nj) if abs(t[m.offset[j]]) > m.tmax[j])
        if kind == "near":
            # a body whose contact bit is set while none of its corners penetrates, before and after the step: only the
            # touching band (-contact_tol < pen <= 0) sets it
            cp, _ = corner_pens(m, o, env, q, qd)
            for b in np.flatnonzero(c):
                if np.all(cp_before[cp_before[:, 0] == b, 4] <= 0) and np.all(cp[cp[:, 0] == b, 4] <= 0):
                    self.c["touching, no force"] += 1

    def check(self, key, kinds=KINDS, skip=()):
        print("coverage %-34s %s" % (key, self.c))
        need = {"vertex": ["vertex slot 3", "vertex past seam"], "limit": ["past limit"], "clamp": ["clamped"], "deep": ["deep corners"], "near": ["touching, no force"],
                "friction": ["slow friction", "fast friction"], "broad": ["in margin"], "seam": ["over seam"]}
        for k in kinds:
            for what in need[k]:
                assert what in skip or self.c[what] > 0, (key, what, self.c)


def stress_rounds(g, o, m, n, rounds, worst, key, seed, steps_after=5, cov=None, kinds=KINDS, shadow=None, sens=None):
    """rounds x n stress states (env e of round r gets kind (r n + e) mod len(kinds)), each followed by steps_after forced steps"""
    rng = np.random.default_rng(seed)
    ints, _ = int_fields(n_params(o), m.nj)
    nout = net_out_size(g, m)
    cov = cov or Coverage()
    drawn = {}
    for r in range(rounds):
        plan = {}
        blown = [e for e in range(n) if not np.abs(o.get_state(e)[1]).max() < 100.0]
        if blown:                      # a stress state that went unstable: both sides reset the env (bit-exact)
            g.Reset(blown)
            for e in blown:
                o.reset(e)
                if sens is not None:
                    sens.o.reset(e)
            cov.c["resets"] += len(blown)
        for e in range(n):
            kind = kinds[(r * n + e) % len(kinds)]
            drawn[kind] = drawn.get(kind, -1) + 1
            q, qd, tau, c = o.get_state(e)
            q, qd, tau = stress_state(kind, drawn[kind], rng, m, o, e, q, qd, tau)
            o.set_state(e, q=q, qd=qd, tau=tau, contact=c)
            plan[e] = (kind, cov.at_install(kind, m, o, e, q, qd))
            if "vertex" in kinds:
                cov.vertices_at_install(m, o, e, q)
        for k in range(steps_after):
            cov.c["model mattered"] += int(step_all(g, o, range(n), shadow, sens))
            compare(g, o, range(n), worst, "%s/%s" % (key, "stress"), (r, k), ints, nout, sens)
            if k == 0:
                for e, (kind, cp) in plan.items():
                    cov.after_step(kind, m, o, e, cp)
    return cov


def translate_forward(m, o, env, ahead, clearance=0.004):
    """the env's state moved along the ground to `ahead` metres short of the point where the ground streams in a new segment
    (the window ends 11 m ahead of the root), its lowest corner `clearance` above the terrain"""
    q, qd, tau, c = o.get_state(env)
    q = q.copy()
    d, mnx, _ = Ground(o, env).segs[1]
    q[0] = mnx + (d.size - 1) * SPACING - 11.0 - ahead
    cp, _ = corner_pens(m, o, env, q, qd)
    i = np.argmax(cp[:, 4])
    return lift_to(q, cp[i, 4], cp[i, 5], -clearance), qd, tau, c


# --------------------------------------------------------------------------------------------------- 2. forced trajectories
TRAJ = [("dog_flat", 600), ("dog_slopes_mixed", 600), ("goat_cliffs", 600), ("raptor_narrow_gaps", 600)]


def run_trajectory(assets, scene, n, steps, worst, seam_envs=4, key=None):
    """n envs, the first seam_envs of them moved to 4 .. 7 cm short of where the ground streams in a new segment"""
    g, o, m = make_pair(assets, scene, n)
    key = key or scene
    for e in range(min(seam_envs, n)):
        q, qd, tau, c = translate_forward(m, o, e, 0.04 + 0.01 * e)
        o.set_state(e, q=q, qd=qd, tau=tau, contact=c)
    mnx0 = [g.GetTerrain(e, 0)[1] for e in range(n)]
    decisions = forced_steps(g, o, m, range(n), steps, worst, key)
    moved = sum(g.GetTerrain(e, 0)[1] != mnx0[e] for e in range(n))
    for e in range(n):
        for s in (0, 1):
            gd, gmx, gfl = g.GetTerrain(e, s)
            od, omx, ofl = o.terrain(e, s)
            assert gmx == omx and gfl == ofl and np.array_equal(gd, od), (scene, e, s)
    return g, o, m, decisions, moved


@pytest.mark.parametrize("scene,steps", TRAJ)
def test_forced_trajectory(assets, scene, steps):
    worst = Worst()
    g, o, m, decisions, moved = run_trajectory(assets, scene, 8, steps, worst)
    print("forced %s: %d decisions, %d envs streamed in a new ground segment" % (scene, decisions, moved))
    worst.report()
    assert decisions >= 8 and moved >= 1


# --------------------------------------------------------------------------------------------------- 3. stress states
STRESS = ["dog_flat", "dog_slopes_mixed", "goat_cliffs", "raptor_narrow_gaps"]


@pytest.mark.parametrize("scene", STRESS)
def test_stress_states(assets, scene):
    n = 8
    worst = Worst()
    g, o, m = make_pair(assets, scene, n)
    sens = Sensitivity(assets, scene, n)
    forced_steps(g, o, m, range(n), 30, worst, scene, sens=sens)
    cov = stress_rounds(g, o, m, n, 4, worst, scene, seed=sum(map(ord, scene)), sens=sens)
    worst.report()
    cov.check(scene)


# --------------------------------------------------------------------------------------------------- 4. the vertex contact model
@pytest.mark.parametrize("scene", ["dog_slopes_mixed", "goat_cliffs", "raptor_narrow_gaps"])
def test_vertex_contact_model(assets, scene, monkeypatch):
    """TRL_VERTEX_CONTACTS=1 on the GPU, ORC_VTX=1 in the oracle: forced trajectory and stress states.  A shadow oracle with the
    corner-only model steps from the same states, to show that the vertex contacts changed the physics."""
    from pyoracle import Oracle
    n = 8
    monkeypatch.setenv("TRL_VERTEX_CONTACTS", "1")
    monkeypatch.setenv("ORC_VTX", "1")
    g, o, m = make_pair(assets, scene, n)
    monkeypatch.delenv("ORC_VTX")
    shadow = Oracle(os.path.join(assets, scene + ".trlpack"), n, 0, terrain_seeds=list(range(101, 101 + n)))
    monkeypatch.setenv("ORC_VTX", "1")
    sens = Sensitivity(assets, scene, n)
    key = scene + "/vertex"
    worst = Worst()
    cov = Coverage()
    for e in range(4):
        q, qd, tau, c = translate_forward(m, o, e, 0.04 + 0.01 * e)
        o.set_state(e, q=q, qd=qd, tau=tau, contact=c)
    mnx0 = [g.GetTerrain(e, 0)[1] for e in range(n)]
    stats = {}
    forced_steps(g, o, m, range(n), 300, worst, key, shadow=shadow, stats=stats, sens=sens)
    assert sum(g.GetTerrain(e, 0)[1] != mnx0[e] for e in range(n)) >= 1
    cov.c["model mattered"] += stats["model mattered"]
    stress_rounds(g, o, m, n, 6, worst, key, seed=7 + sum(map(ord, scene)), cov=cov, kinds=KINDS + ("vertex", "vertex"),
                  shadow=shadow, sens=sens)
    worst.report()
    cov.check(key, KINDS + ("vertex",))
    assert cov.c["model mattered"] >= 20, cov.c


# --------------------------------------------------------------------------------------------------- 5. launch shapes
def shape_states(m, o, n, special, seed):
    """env states for a batch with one terrain: the same stress state at the `special` envs, distinct perturbations elsewhere"""
    rng = np.random.default_rng(seed)
    q0, qd0, tau0, c0 = o.get_state(0)
    sq, sqd, stau = stress_state("deep", 0, np.random.default_rng(seed + 1), m, o, 0, q0, qd0, tau0)
    sq, sqd, stau = stress_state("limit", 0, np.random.default_rng(seed + 2), m, o, 0, sq, sqd + 0.3, stau)
    out = []
    for e in range(n):
        if e in special:
            out.append((sq, sqd, stau, c0))
            continue
        q, qd = q0.copy(), qd0.copy()
        q[0] += rng.uniform(-0.03, 0.03)
        q[2:] += rng.normal(0.0, 0.05, q.size - 2)
        qd += rng.normal(0.0, 0.5, qd.size)
        out.append((q, qd, rng.normal(0.0, 20.0, qd.size) * (np.arange(qd.size) >= 3), c0))
    return out


def env_result(g, e, nout):
    q, qd, tau, c = g.GetState(e)
    r = [q, qd, tau, c, g.GetCtrl(e), g.GetPoliState(e)]
    if nout:
        r.append(g.GetNetOut(e, nout))
    return r


def run_shape(assets, scene, n, seed=5, tol=TOL, ref=None):
    from pyoracle import Oracle
    import deepterrainrl_b200 as trl
    pack = os.path.join(assets, scene + ".trlpack")
    m = Model(pack)
    g = trl.ScenarioPoliEval(pack, n, terrain_seeds=[77] * n)
    o = Oracle(pack, n, 0, terrain_seeds=[77] * n)
    tail = max([e for e in range(n) if e % 4 == 3] or [0])
    special = sorted({0, n - 1, tail})
    states = shape_states(m, o, n, special, seed)
    for e, (q, qd, tau, c) in enumerate(states):
        g.SetState(e, q=q, qd=qd, tau=tau, contact=c)
        o.set_state(e, q=q, qd=qd, tau=tau, contact=c)
    g.EnvStep(H)
    for e in range(n):
        o.env_step(e, H)
    worst = Worst(tol)
    ints, _ = int_fields(n_params(o), m.nj)
    nout = net_out_size(g, m)
    decided = compare(g, o, range(n), worst, "%s n=%d" % (scene, n), 0, ints, nout)
    assert len(decided) == n                     # the first step after a reset decides
    ref = ref if ref is not None else env_result(g, special[0], nout)
    for e in special:
        got = env_result(g, e, nout)
        assert all(np.array_equal(a, b) for a, b in zip(got, ref)), (n, e)
    g.close()
    return worst, ref


def test_launch_shapes_are_batch_invariant(assets):
    """one env per warp, 4 warps per CTA: the same state at env 0, at the last env and at a CTA tail gives bit-identical results
    at every batch size, and every distinct state matches the oracle"""
    ref = None
    for n in (1, 3, 5, 129, 4097):
        worst, ref = run_shape(assets, "dog_slopes_mixed", n, ref=ref)
        worst.report()


# --------------------------------------------------------------------------------------------------- 6. one Update from forced states
def fallen_state(m, o, e, how):
    q, qd, tau, c = o.get_state(e)
    q, qd = q.copy(), qd.copy()
    if how == "tilt":
        q[2] = 0.9 * np.pi              # past the fall test |root angle| > 0.8 pi
        qd[2] = 0.0
    else:                               # torso on the ground
        q[2] = 0.5 * np.pi
    cp, _ = corner_pens(m, o, e, q, qd)
    i = np.argmax(cp[:, 4])
    return lift_to(q, cp[i, 4], cp[i, 5], 0.002), qd, tau, c


def run_update(assets, scene, n, monkeypatch, env, mode=0, tol=1e-9, forced=None):
    from pyoracle import Oracle
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    g, o, m = make_pair(assets, scene, n, mode=mode)
    # the state every env returns to at a reset (the same terrain seed gives the same ground and starting height)
    fresh = Oracle(os.path.join(assets, scene + ".trlpack"), n, mode, terrain_seeds=list(range(101, 101 + n)))
    start = [fresh.get_state(e)[:2] for e in range(n)]
    del fresh
    for k in env:
        monkeypatch.delenv(k)
    if mode:
        g.EnableExplore(1, 0.2, 0.025, 0.01)
        o.set_explore(1, 0.2, 0.025, 0.01)
    worst = Worst(tol)
    # exploration: long enough for every env to have finished two gait cycles, so that tuples are recorded
    forced_steps(g, o, m, range(n), forced or (300 if mode else 40), worst, scene)
    for e, how in ((1, "tilt"), (n - 1, "tilt"), (2, "torso")):
        q, qd, tau, c = fallen_state(m, o, e, how)
        o.set_state(e, q=q, qd=qd, tau=tau, contact=c)
    force(g, o, range(n))
    g.Update(1.0 / 30.0)
    g.Sync()
    o.update(1.0 / 30.0, threads=8)
    ints, _ = int_fields(n_params(o), m.nj)
    key = "%s update %s%s" % (scene, ",".join("%s=%s" % kv for kv in env.items()) or "overlapped", " explore" if mode else "")
    is_start = lambda q, qd, e: np.array_equal(q, start[e][0]) and np.array_equal(qd, start[e][1])
    o_reset = [e for e in range(n) if is_start(*o.get_state(e)[:2], e)]
    g_reset = [e for e in range(n) if is_start(*g.GetState(e)[:2], e)]
    assert 1 in o_reset and n - 1 in o_reset, o_reset        # the tilted envs fell and were reset
    assert g_reset == o_reset, (g_reset, o_reset)            # the same envs, the torso-down env 2 included or not on both sides
    for e in range(n):
        gq, gqd, gt, gc = g.GetState(e)
        oq, oqd, ot, oc = o.get_state(e)
        if e in o_reset:                # reset after the fall: bit-exact
            worst.exact(key, "reset q", gq, oq, e)
            worst.exact(key, "reset qd", gqd, oqd, e)
        worst.rel(key, "q", gq, oq, e)
        worst.rel(key, "qd", gqd, oqd, e)
        worst.rel(key, "tau", gt, ot, e)
        worst.exact(key, "contact", gc, oc, e)
        gk, ok = g.GetCtrl(e), o.get_ctrl(e)
        dbl = np.ones(ok.size, bool)
        dbl[ints] = False
        worst.rel(key, "ctrl", gk[dbl], ok[dbl], e)
        worst.exact(key, "ctrl ints", gk[ints], ok[ints], e)
    gs, os_ = g._stats(), o.eval_stats()
    assert (gs["cycles"], gs["episodes"], gs["steps"]) == (os_["cycles"], os_["episodes"], os_["steps"]), (gs, os_)
    if not mode:
        assert os_["episodes"] >= 2
        gd, ge = g.GetDistLog()
        for e in range(n):
            od = o.dist_log(e)
            worst.rel(key, "dist log", gd[ge == e], od, e)
            assert (ge == e).sum() == od.size
    else:
        gr, gf, ge = g.GetTuples(f64=True)
        orr, of, oe = o.tuples()
        assert gr.shape == orr.shape and gr.shape[0] > 0, (gr.shape, orr.shape, np.bincount(ge, minlength=n), np.bincount(oe, minlength=n))
        gi, oi = np.argsort(ge, kind="stable"), np.argsort(oe, kind="stable")
        worst.exact(key, "tuple env", ge[gi], oe[oi], "tuples")
        worst.exact(key, "tuple flags", gf[gi], of[oi], "tuples")
        worst.rel(key, "tuples", gr[gi], orr[oi], "tuples")
    return worst


@pytest.mark.parametrize("env", [{}, {"TRL_SERIAL_SCHEDULE": "1"}, {"TRL_GROUPS": "3"}], ids=["overlapped", "serial", "groups3"])
@pytest.mark.parametrize("mode", [0, 1], ids=["eval", "explore"])
def test_update_from_forced_states(assets, monkeypatch, env, mode):
    """one Update(1/30) (captured graph, catch-up launches, env groups, end-of-update resets) from forced states, fallen envs
    among them; 40 envs leave a ragged third group of 8"""
    worst = run_update(assets, "dog_slopes_mixed", 40, monkeypatch, env, mode=mode)
    worst.report()
