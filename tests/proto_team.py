#!/usr/bin/env python
"""float64 numpy restatement of the ARTICULATION substep of csrc/rollout_team.cu for TREES, written the way the kernel computes it --
world frames / velocities / accelerations by pointer jumping over the ancestors, composites as differences of suffix sums over the
depth-first body order, joint-space LDL^T with the leaves eliminated first -- and checked against the oracle (body-frame ABA with
dense 6x6 transforms) on the host; and of its contact solve over generalised coordinates (a free box on the ground: linear + BODY-axis
angular velocity components with scalar inverse inertias, cached rows) against the oracle's world-frame solve; and of the WHOLE step of
the push scenes (articulation + contacts in the oracle's order up to the capacity + Gauss-Seidel over joints and free-body components)
in lock-step with the oracle.  Formulation checks that need no GPU (tests/test_proto_team.py runs them):

    python tests/proto_team.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from proto_lanes import q2R, qmul, qrot, sym  # noqa: E402


def tree_tables(parent, G):
    """What the kernel keeps per lane: jump[r][i] = the 2^r-th ancestor of body i (-1: none), desc[i] = set of i and its descendants,
    end[i] = first body after the subtree of i (depth-first numbering: the subtree is the index range [i, end))."""
    nb = len(parent)
    R = {4: 2, 8: 3, 16: 4}[G]
    jump = [list(parent)]
    for r in range(1, R):
        jump.append([jump[r - 1][jump[r - 1][i]] if jump[r - 1][i] >= 0 else -1 for i in range(nb)])
    anc = [{i} for i in range(nb)]
    for r in range(R):
        anc = [anc[i] | (anc[jump[r][i]] if jump[r][i] >= 0 else set()) for i in range(nb)]
    desc = [{j for j in range(nb) if i in anc[j]} for i in range(nb)]
    end = [i + len(desc[i]) for i in range(nb)]
    for i in range(nb):
        assert desc[i] == set(range(i, end[i])), "bodies must be numbered depth first"
        assert len(anc[i]) <= 2 ** R, "tree deeper than the team is wide"
    return jump, desc, end


def anc_sum(x, jump):
    """x[i] <- sum of x over i and its ancestors (pointer jumping: after round r every entry covers 2^(r+1) bodies up the tree)"""
    x = [np.array(v, float) for v in x]
    for jr in jump:
        x = [x[i] + x[jr[i]] if jr[i] >= 0 else x[i] for i in range(len(x))]
    return x


def subtree_sum(x, end):
    """x[i] <- sum over the subtree of i = suffix sum at i minus suffix sum at the subtree's end"""
    P = np.cumsum(np.array(x, float)[::-1], axis=0)[::-1]
    return [P[i] - (P[end[i]] if end[i] < len(x) else 0.0) for i in range(len(x))]


def rollout(m, p, state0, actions_k, want_pivots=False, contact_cb=None):
    """actions_k: (T, nu) of ONE rollout; returns (q, qd) after T steps [and the LDL pivots of the last substep].
    contact_cb(R, origins, Sn, Sf, vp, pivots, h) -> corrected joint velocities: the contact phase, called once per substep with what
    the articulation phase hands over (frames, motion subspaces, predicted velocities, the articulated-body diagonals)."""
    nb, T = m.nb, p.T
    G = 8 if nb <= 8 else 16
    h = p.dt / p.substeps
    vel = m.drive_mode == 0
    parent = [m.parent[i] for i in range(nb)]
    jump, desc, end = tree_tables(parent, G)
    q, qd = np.array(state0[:nb], float), np.array(state0[nb:2 * nb], float)
    bq, bp = np.array(m.base_quat[:], float), np.array(m.base_pos[:], float)
    a0f = -np.array(m.gravity[:], float) if m.gravity_on else np.zeros(3)
    tq = [np.array(m.tree_quat[i][:], float) for i in range(nb)]
    tp = [np.array(m.tree_p[i][:], float) for i in range(nb)]
    tR = [np.array(m.tree_R[i][:], float).reshape(3, 3) for i in range(nb)]
    rev = [m.jtype[i] == 0 for i in range(nb)]
    tax = [np.zeros(3) if rev[i] else tR[i][:, 2] for i in range(nb)]
    for i in range(nb):
        if parent[i] < 0:       # the base pose is folded into every root body's parent transform
            tp[i] = bp + qrot(bq, tp[i]); tax[i] = qrot(bq, tax[i]); tq[i] = qmul(bq, tq[i])
    mass = np.array(m.mass[:nb], float)
    com = [np.array(m.mcom[i][:], float) / mass[i] if mass[i] > 0 else np.zeros(3) for i in range(nb)]
    Ic = []
    for i in range(nb):
        c = com[i]
        Ic.append(sym(np.array(m.inertia[i][:], float)) - mass[i] * (c @ c * np.eye(3) - np.outer(c, c)))
    mc = subtree_sum(list(mass), end)
    pivots = None
    for t in range(T):
        u = actions_k[t] * p.u_scale
        tgt0 = np.array([m.cmd_c0[i] * u[m.cmd_i0[i]] + m.cmd_c1[i] * u[m.cmd_i1[i]] for i in range(nb)])
        for _ in range(p.substeps):
            tgt = tgt0.copy()
            if m.planar_base:   # body twist (v, omega) -> world-frame velocity targets of the three virtual joints
                sy, cy = np.sin(q[2]), np.cos(q[2])
                tgt[0] = u[0] * (m.fwd_axis[0] * cy - m.fwd_axis[1] * sy)
                tgt[1] = u[0] * (m.fwd_axis[0] * sy + m.fwd_axis[1] * cy)
                tgt[2] = u[1]
            # frames: product of the local transforms along the path from the root, by pointer jumping
            ql, pl = [], []
            for i in range(nb):
                ang = 0.5 * q[i] * (1.0 if rev[i] else 0.0)
                ql.append(qmul(tq[i], np.array([0, 0, np.sin(ang), np.cos(ang)])))
                pl.append(tp[i] + q[i] * tax[i])
            for jr in jump:
                nq, npos = list(ql), list(pl)
                for i in range(nb):
                    if jr[i] >= 0:
                        npos[i] = pl[jr[i]] + qrot(ql[jr[i]], pl[i]); nq[i] = qmul(ql[jr[i]], ql[i])
                ql, pl = nq, npos
            R = [q2R(x) for x in ql]
            Sn, Sf = [], []
            for i in range(nb):
                ax = R[i][:, 2]
                Sn.append(ax if rev[i] else np.zeros(3)); Sf.append(np.cross(pl[i], ax) if rev[i] else ax)
            Vn = anc_sum([qd[i] * Sn[i] for i in range(nb)], jump)
            Vf = anc_sum([qd[i] * Sf[i] for i in range(nb)], jump)
            A, hw, fn, ff_, an, af = [], [], [], [], [], []
            for i in range(nb):
                cw = pl[i] + R[i] @ com[i]
                hwi = mass[i] * cw
                Ai = R[i] @ Ic[i] @ R[i].T + (hwi @ cw) * np.eye(3) - np.outer(hwi, cw)
                w, v = Vn[i], Vf[i]
                nn = Ai @ w + np.cross(hwi, v)
                ff = mass[i] * v - np.cross(hwi, w)
                fn.append(np.cross(w, nn) + np.cross(v, ff)); ff_.append(np.cross(w, ff))
                an.append(np.cross(w, qd[i] * Sn[i])); af.append(np.cross(w, qd[i] * Sf[i]) + np.cross(v, qd[i] * Sn[i]))
                A.append(Ai); hw.append(hwi)
            an = anc_sum(an, jump); af = [x + a0f for x in anc_sum(af, jump)]
            for i in range(nb):
                fn[i] = fn[i] + A[i] @ an[i] + np.cross(hw[i], af[i])
                ff_[i] = ff_[i] + mass[i] * af[i] - np.cross(hw[i], an[i])
            Ac, hc, fcn, fcf = subtree_sum(A, end), subtree_sum(hw, end), subtree_sum(fn, end), subtree_sum(ff_, end)
            Fn = [Ac[i] @ Sn[i] + np.cross(hc[i], Sf[i]) for i in range(nb)]
            Ff = [mc[i] * Sf[i] - np.cross(hc[i], Sn[i]) for i in range(nb)]
            bias = np.array([Sn[i] @ fcn[i] + Sf[i] @ fcf[i] for i in range(nb)])
            M = np.zeros((nb, nb))   # M[r, j] = F_r . S_j for the descendants r of j (and symmetric), 0 between different branches
            for j in range(nb):
                for r in desc[j]:
                    M[r, j] = M[j, r] = Fn[r] @ Sn[j] + Ff[r] @ Sf[j]
            sat = np.zeros(nb)
            for solve in range(2):
                tau, dimp = np.zeros(nb), np.zeros(nb)
                for i in range(nb):
                    kd, b, arm, eff = m.kd[i], m.damping[i], m.armature[i], m.effort[i]
                    if sat[i] != 0:
                        tau[i] = sat[i] * eff - b * qd[i]; dimp[i] = arm + h * b
                    elif vel:
                        tau[i] = kd * (tgt[i] - qd[i]) - b * qd[i]; dimp[i] = arm + h * (kd + b)
                    else:
                        tau[i] = min(max(tgt[i], -eff), eff) - (kd + b) * qd[i]; dimp[i] = arm + h * (kd + b)
                # LDL^T in REVERSED body order (virtual index nb - 1 - body: leaves first), as the kernel runs it
                perm = np.arange(nb)[::-1]
                Hv = (M + np.diag(dimp))[np.ix_(perm, perm)]
                yv = (tau - bias)[perm]
                L, D = np.eye(nb), np.zeros(nb)
                Hw = Hv.copy()
                for kk in range(nb):
                    D[kk] = Hw[kk, kk]
                    L[kk + 1:, kk] = Hw[kk + 1:, kk] / D[kk]
                    Hw[kk + 1:, kk + 1:] -= np.outer(L[kk + 1:, kk], Hw[kk, kk + 1:])
                z = np.linalg.solve(L, yv) / D
                qdd = np.linalg.solve(L.T, z)[perm]           # back to body order (perm is its own inverse)
                pivots = D[perm]
                if solve == 0 and vel:
                    td = np.array([m.kd[i] * (tgt[i] - (qd[i] + h * qdd[i])) for i in range(nb)])
                    newly = np.abs(td) > np.array(m.effort[:nb])
                    if not newly.any():
                        break
                    sat = np.where(newly, np.sign(td), 0.0)
                else:
                    break
            vj = qd + h * qdd
            if contact_cb is not None:
                vj = contact_cb(R, pl, Sn, Sf, vj, pivots, h)
            for i in range(nb):
                vn = min(max(vj[i], -m.qd_max[i]), m.qd_max[i])
                x = q[i] + h * vn
                if x < m.q_lo[i]:
                    x = m.q_lo[i]; vn = max(vn, 0.0)
                if x > m.q_hi[i]:
                    x = m.q_hi[i]; vn = min(vn, 0.0)
                q[i], qd[i] = x, vn
    return (q, qd, pivots) if want_pivots else (q, qd)


def aba_diagonals(m, p, q, tgt_dimp):
    """D_j of the articulated-body recursion (world frame, spatial quantities about the world origin) for the configuration q:
    what the contact solve uses as joint compliance -- computed independently of the LDL^T above (6x6 articulated inertias)."""
    nb = m.nb
    parent = [m.parent[i] for i in range(nb)]
    bq, bp = np.array(m.base_quat[:], float), np.array(m.base_pos[:], float)
    Rw, ow = [None] * nb, [None] * nb
    S = [None] * nb
    IA = [None] * nb
    for i in range(nb):
        Rp, op = (q2R(bq), bp) if parent[i] < 0 else (Rw[parent[i]], ow[parent[i]])
        Rt = Rp @ np.array(m.tree_R[i][:], float).reshape(3, 3)
        oi = op + Rp @ np.array(m.tree_p[i][:], float)
        ax = Rt[:, 2]
        if m.jtype[i] == 0:
            c, s = np.cos(q[i]), np.sin(q[i])
            Rw[i] = Rt @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]]); ow[i] = oi
            S[i] = np.concatenate([ax, np.cross(oi, ax)])
        else:
            Rw[i] = Rt; ow[i] = oi + q[i] * ax
            S[i] = np.concatenate([np.zeros(3), ax])
        mass = m.mass[i]
        com = np.array(m.mcom[i][:], float) / mass if mass > 0 else np.zeros(3)
        Io = sym(np.array(m.inertia[i][:], float))
        Icm = Io - mass * (com @ com * np.eye(3) - np.outer(com, com))
        cw = ow[i] + Rw[i] @ com
        cx = np.array([[0, -cw[2], cw[1]], [cw[2], 0, -cw[0]], [-cw[1], cw[0], 0]])
        I6 = np.zeros((6, 6))     # spatial inertia about the world origin, [angular; linear] ordering
        I6[:3, :3] = Rw[i] @ Icm @ Rw[i].T - mass * cx @ cx
        I6[:3, 3:] = mass * cx
        I6[3:, :3] = -mass * cx
        I6[3:, 3:] = mass * np.eye(3)
        IA[i] = I6
    D = np.zeros(nb)
    for i in range(nb - 1, -1, -1):
        U = IA[i] @ S[i]
        D[i] = S[i] @ U + tgt_dimp[i]
        if parent[i] >= 0:
            IA[parent[i]] = IA[parent[i]] + IA[i] - np.outer(U, U) / D[i]
    return D


def check(names=("panda_gripper", "omnipanda", "albert", "jackal", "boxer"), K=3, T=6, verbose=True):
    from oracle import oracle as orc
    from scenes import robot_setup
    links = {"albert": "mmrobot_link7", "omnipanda": "panda_hand", "jackal": "ee_link", "boxer": "ee_link", "panda_gripper": "panda_hand"}
    worst_all = 0.0
    for name in names:
        sc, p, state0 = robot_setup(name, links[name], K=K, T=T, u_lim=0.4)
        rng = np.random.default_rng(4)
        actions = rng.uniform(-0.4, 0.4, (T, sc.nu, K)).astype(np.float32)
        actions[:, :, 0] *= 6.0                                  # one rollout far beyond the effort limits -> saturation re-solve
        st_ref, _ = orc.rollout(sc.model, p, state0, actions, use_double=True, root0=sc.root_state0.astype(np.float32))
        nb = sc.model.nb
        worst = 0.0
        for k in range(K):
            q, qd, piv = rollout(sc.model, p, state0, actions[:, :, k].astype(float), want_pivots=True)
            worst = max(worst, np.abs(q - st_ref[:nb, k]).max(), np.abs(qd - st_ref[nb:2 * nb, k]).max() * 1e-2)
        # the leaves-first pivots ARE the articulated-body diagonals D_j (joint compliance of the contact solve); unsaturated drive terms
        h = p.dt / p.substeps
        dimp = np.array([sc.model.armature[i] + h * (sc.model.kd[i] + sc.model.damping[i]) for i in range(nb)])
        q0 = np.array(state0[:nb], float)
        _, _, piv0 = rollout(sc.model, _one_substep(p), state0, np.zeros((1, sc.nu)), want_pivots=True)
        D = aba_diagonals(sc.model, p, q0, dimp)
        dpiv = np.abs(piv0 / D - 1.0).max()
        if verbose:
            print(f"{name:14s} nb = {nb:2d}: max |q - oracle| (and 1e-2 |qd - oracle|) over {K} rollouts, T = {T}: {worst:.3e};  max |pivot / D_j - 1| = {dpiv:.2e}")
        assert worst < 5e-5, (name, worst)
        assert dpiv < 1e-6, (name, dpiv)      # (the model block holds tree_R and tree_quat as separately rounded float32)
        worst_all = max(worst_all, worst)
    return worst_all


def _one_substep(p):
    import copy
    p1 = copy.copy(p)
    p1.T, p1.substeps, p1.dt = 1, 1, p.dt / p.substeps
    return p1




def ground_corners(R, c, half, margin):
    """Ground points of a box (rotation R, centre c), in corner-index order: the corners among the 4 lowest of the 8 (ties by corner
    index) that lie below `margin`."""
    pts = [R @ (np.array([ix, iy, iz]) * half) + c for ix in (-1, 1) for iy in (-1, 1) for iz in (-1, 1)]
    z = [p[2] for p in pts]
    rank = [sum(z[o] < z[k] or (z[o] == z[k] and o < k) for o in range(8)) for k in range(8)]
    return [pts[k] for k in range(8) if rank[k] < 4 and z[k] < margin]


# ------------------------------------------------------------------------------------------------------------------------------
# The contact solve of rollout_team.cu in GENERALISED COORDINATES, for the part that is new against the oracle: a free body's three
# linear velocity components (world) and three angular velocity components IN BODY AXES, one scalar inverse inertia each, contact rows
# cached once per substep.  Case: a free box on the ground plane (up to 4 corner contacts), one model step of the heijn_push scene with
# the robot far away -- the oracle solves it with world-frame inverse inertia tensors and point velocities.
def free_box_step(m, p, box_state, f=0):
    """One model step of free body f alone on the ground (no other contact partner in reach); box_state = its 13 root-state numbers.
    Returns the 13 numbers after the step."""
    h = p.dt / p.substeps
    x, qt, v, w = (np.array(box_state[0:3], float), np.array(box_state[3:7], float), np.array(box_state[7:10], float),
                   np.array(box_state[10:13], float))
    shape = next(s for s in range(m.nshapes) if m.shape_owner_kind[s] == 2 and m.shape_owner[s] == f)
    half = np.array(m.free_half[f][:], float)
    mass = float(m.free_mass[f])
    Iinv = 1.0 / (mass / 3.0 * np.array([half[1] ** 2 + half[2] ** 2, half[0] ** 2 + half[2] ** 2, half[0] ** 2 + half[1] ** 2]))
    minv = np.concatenate([np.full(3, 1.0 / mass), Iinv])                      # one scalar inverse inertia per coordinate
    kp, kd = float(m.contact_kp), float(m.contact_kd)
    gamma, beta = 1.0 / (h * (h * kp + kd)), h * kp / (h * kp + kd)
    mu = 0.5 * (float(m.shape_friction[shape]) + float(m.ground_friction))
    g = np.array(m.gravity[:], float)
    for _ in range(p.substeps):
        R = q2R(qt)
        sq, sp = np.array(m.shape_quat[shape][:], float), np.array(m.shape_pos[shape][:], float)
        Rs, cs = R @ q2R(sq), x + R @ sp
        contacts = [(pt, -pt[2]) for pt in ground_corners(Rs, cs, half, float(m.ground_margin))]
        if m.free_gravity[f]:
            v = v + h * g
        u = np.concatenate([v, R.T @ w])                                       # generalised velocities: world linear, BODY-axis angular
        n = np.array([0.0, 0.0, 1.0])
        e = np.array([1.0, 0, 0]) if abs(n[0]) < 0.9 else np.array([0, 1.0, 0])
        t1 = np.cross(n, e); t1 /= np.linalg.norm(t1); t2 = np.cross(n, t1)
        rows, consts, lam = [], [], []
        for pt, d in contacts:                                                 # once per contact: rows, inverse effective masses, bias
            r = pt - x
            J = [np.concatenate([dr, R.T @ np.cross(r, dr)]) for dr in (n, t1, t2)]
            k = [float((Jr * Jr) @ minv) for Jr in J]
            bias = min(beta * d / h, float(m.max_depen)) if d > 0 else d / h
            rows.append(J)
            consts.append((bias, 1.0 / (k[0] + gamma) if k[0] > 1e-9 else 0.0, 1.0 / k[1] if k[1] > 1e-9 else 0.0, 1.0 / k[2] if k[2] > 1e-9 else 0.0))
            lam.append(np.zeros(3))
        for _it in range(m.contact_iters):
            for c, J in enumerate(rows):
                bias, ikn, ikt1, ikt2 = consts[c]
                if not ikn > 0:
                    continue
                vn, v1, v2 = (float(Jr @ u) for Jr in J)
                ln, lt1, lt2 = lam[c]
                ln_new = max(0.0, ln + (-vn + bias - gamma * ln) * ikn)
                lim = mu * ln_new
                lt1_new = min(max(lt1 - v1 * ikt1, -lim), lim) if ikt1 > 0 else lt1
                lt2_new = min(max(lt2 - v2 * ikt2, -lim), lim) if ikt2 > 0 else lt2
                u = u + minv * (J[0] * (ln_new - ln) + J[1] * (lt1_new - lt1) + J[2] * (lt2_new - lt2))
                lam[c] = np.array([ln_new, lt1_new, lt2_new])
        v, w = u[:3], R @ u[3:]
        x = x + h * v
        wq = np.array([w[0], w[1], w[2], 0.0])
        qt = qt + 0.5 * h * qmul(wq, qt)
        qt = qt / np.linalg.norm(qt)
    return np.concatenate([x, qt, v, w])


def check_free_box(verbose=True):
    from oracle import oracle as orc
    from scenes import push_setup
    sc, p, s0 = push_setup(K=4, T=2, obstacles=False, block_pos=(3.0, -2.0, 0.1), robot_pos=(0.0, 1.5, 0.05))
    m = sc.model
    nd2 = 2 * sc.ndof
    NS = orc.lib().oracle_state_size(__import__("ctypes").byref(m))
    rng = np.random.default_rng(12)
    worst = 0.0
    for trial in range(6):
        ang = rng.uniform(-0.04, 0.04, 3)                                      # a slightly tilted box, some corners in the ground, some above it
        qt = np.array([np.sin(ang[0] / 2), 0, 0, np.cos(ang[0] / 2)])
        qt = qmul(np.array([0, np.sin(ang[1] / 2), 0, np.cos(ang[1] / 2)]), qt)
        qt = qmul(np.array([0, 0, np.sin(0.7 + ang[2]), np.cos(0.7 + ang[2])]), qt)
        half = np.array(m.free_half[0][:], float)
        box = np.concatenate([[3.0, -2.0, half[2] - 0.002 * trial], qt, rng.uniform(-0.5, 0.5, 3) * [1, 1, 0.2], rng.uniform(-1.0, 1.0, 3)])
        state = np.zeros((NS, p.K), np.float32)
        state[:nd2] = s0[:, None]
        state[nd2:nd2 + 13] = box.astype(np.float32)[:, None]
        box32 = state[nd2:nd2 + 13, 0].astype(float)                          # (the state rows are float32: start both from the same numbers)
        ref, _ = orc.rollout(m, p, None, np.zeros((p.T, sc.nu, p.K), np.float32), 0, 1, state=state.copy(), root0=sc.root_state0, want_obs=False, use_double=True)
        mine = free_box_step(m, p, box32)
        err = np.abs(mine - ref[nd2:nd2 + 13, 0]).max()
        moved = np.abs(ref[nd2 + 7:nd2 + 13, 0] - box32[7:13]).max()
        assert moved > 1e-2, "the contacts must have done something"
        worst = max(worst, err)
    if verbose:
        print(f"free box on the ground, generalised-coordinate Gauss-Seidel vs the oracle's world-frame solve, 6 poses: max |state difference| = {worst:.2e}")
    assert worst < 5e-6, worst
    return worst




# ------------------------------------------------------------------------------------------------------------------------------
# The WHOLE step of a contact scene the way rollout_team.cu computes it (articulation above + this contact phase): world shapes,
# contacts in the oracle's order (ground corners; free shape vs every other body's shapes; link shapes vs static shapes; 26 sample
# points of one box inside the other, both directions; capacity max_contacts), Gauss-Seidel over generalised coordinates = the joints
# and, per free body, 3 linear + 3 body-axis angular components.  Boxes only (the shipped push scenes).
def make_contact_phase(m, p, root0, free):
    """free: list of 13-number arrays (pos, quat xyzw, v, w), updated in place every substep.  Returns the contact_cb of rollout()."""
    nb, ns = m.nb, m.nshapes
    parent = [m.parent[i] for i in range(nb)]
    anc = []
    for i in range(nb):
        a, j = set(), i
        while j >= 0:
            a.add(j); j = parent[j]
        anc.append(a)
    half = [np.array(m.shape_half[s][:], float) for s in range(ns)]
    mu_s = [float(m.shape_friction[s]) for s in range(ns)]
    kind = [m.shape_owner_kind[s] for s in range(ns)]           # 0 static, 1 link, 2 free
    own = [m.shape_owner[s] for s in range(ns)]
    for s in range(ns):
        assert m.shape_type[s] == 0, "boxes only"

    def ref(s):
        if kind[s] == 2:
            return ("f", own[s])
        if kind[s] == 1 and own[s] >= 0:
            return ("j", own[s])
        return None

    kp, kd = float(m.contact_kp), float(m.contact_kd)
    mg = float(m.contact_margin)

    def contact_cb(R, o, Sn, Sf, vp, piv, h):
        gamma, beta = 1.0 / (h * (h * kp + kd)), h * kp / (h * kp + kd)
        Rf = [q2R(f[3:7]) for f in free]
        Rs, cs = [], []
        for s in range(ns):
            if kind[s] == 0:
                rs = np.array(root0[m.shape_actor[s]], float)
                Ro, po = q2R(rs[3:7]), rs[0:3]
            elif kind[s] == 1:
                Ro, po = (R[own[s]], o[own[s]]) if own[s] >= 0 else (q2R(np.array(m.base_quat[:], float)), np.array(m.base_pos[:], float))
            else:
                Ro, po = Rf[own[s]], free[own[s]][0:3]
            Rs.append(Ro @ q2R(np.array(m.shape_quat[s][:], float))); cs.append(po + Ro @ np.array(m.shape_pos[s][:], float))
        contacts = []

        def add(ra, rb, pt, n, d, mu):
            if len(contacts) < m.max_contacts:
                contacts.append((ra, rb, np.array(pt), np.array(n), d, mu))

        def points_in_box(a, b, flip):
            cl = Rs[b].T @ (cs[a] - cs[b])
            out = [abs(cl[k]) > half[b][k] for k in range(3)]
            if not any(out):
                out = [True, True, True]
            mu = 0.5 * (mu_s[a] + mu_s[b])
            for idx in range(27):
                if idx == 13:
                    continue
                loc = np.array([idx // 9 - 1, (idx // 3) % 3 - 1, idx % 3 - 1]) * half[a]
                pt = Rs[a] @ loc + cs[a]
                x = Rs[b].T @ (pt - cs[b])
                pen = half[b] - np.abs(x)
                if not all(pen + mg > 0):
                    continue
                ax, best = -1, 0.0
                for k in range(3):
                    if out[k] and (ax < 0 or pen[k] < best):
                        ax, best = k, pen[k]
                n = (1.0 if x[ax] >= 0 else -1.0) * Rs[b][:, ax]
                if not flip:
                    add(ref(a), ref(b), pt, n, best, mu)
                else:
                    add(ref(b), ref(a), pt, -n, best, mu)

        for a in range(ns):
            if kind[a] != 2:
                continue
            if m.ground_plane:
                mu = 0.5 * (mu_s[a] + float(m.ground_friction))
                for pt in ground_corners(Rs[a], cs[a], half[a], float(m.ground_margin)):
                    add(ref(a), None, pt, [0, 0, 1.0], -pt[2], mu)
            for b in range(ns):
                if b == a or ref(b) == ref(a) or (kind[b] == 2 and b < a):
                    continue
                points_in_box(a, b, False); points_in_box(b, a, True)
        for a in range(ns):
            if kind[a] != 1 or ref(a) is None:
                continue
            for b in range(ns):
                if kind[b] == 0:
                    points_in_box(a, b, False); points_in_box(b, a, True)
        g = np.array(m.gravity[:], float)
        for f in range(len(free)):
            if m.free_gravity[f]:
                free[f][7:10] += h * g
        # generalised coordinates: joints, then per free body [v (world); omega (body axes)]
        nco = nb + 6 * len(free)
        u = np.zeros(nco); minv = np.zeros(nco)
        u[:nb] = vp; minv[:nb] = 1.0 / np.maximum(piv, 1e-6)
        for f in range(len(free)):
            hf = np.array(m.free_half[f][:], float); mass = float(m.free_mass[f])
            u[nb + 6 * f:nb + 6 * f + 3] = free[f][7:10]; u[nb + 6 * f + 3:nb + 6 * f + 6] = Rf[f].T @ free[f][10:13]
            minv[nb + 6 * f:nb + 6 * f + 3] = 1.0 / mass
            minv[nb + 6 * f + 3:nb + 6 * f + 6] = 1.0 / (mass / 3.0 * np.array([hf[1] ** 2 + hf[2] ** 2, hf[0] ** 2 + hf[2] ** 2, hf[0] ** 2 + hf[1] ** 2]))
        rows, consts, lam = [], [], []
        for ra, rb, pt, n, d, mu in contacts:
            e = np.array([1.0, 0, 0]) if abs(n[0]) < 0.9 else np.array([0, 1.0, 0])
            t1 = np.cross(n, e); t1 /= np.linalg.norm(t1); t2 = np.cross(n, t1)
            J = []
            for dr in (n, t1, t2):
                Jr = np.zeros(nco)
                for sg, r in ((1.0, ra), (-1.0, rb)):
                    if r is None:
                        continue
                    if r[0] == "j":
                        for j in anc[r[1]]:
                            Jr[j] = sg * (Sf[j] @ dr + Sn[j] @ np.cross(pt, dr))
                    else:
                        f = r[1]
                        Jr[nb + 6 * f:nb + 6 * f + 3] = sg * dr
                        Jr[nb + 6 * f + 3:nb + 6 * f + 6] = sg * (Rf[f].T @ np.cross(pt - free[f][0:3], dr))
                J.append(Jr)
            k = [float((Jr * Jr) @ minv) for Jr in J]
            bias = min(beta * d / h, float(m.max_depen)) if d > 0 else d / h
            rows.append(J); lam.append(np.zeros(3))
            consts.append((bias, mu, 1.0 / (k[0] + gamma) if k[0] > 1e-9 else 0.0, 1.0 / k[1] if k[1] > 1e-9 else 0.0, 1.0 / k[2] if k[2] > 1e-9 else 0.0))
        for _it in range(m.contact_iters):
            for c, J in enumerate(rows):
                bias, mu, ikn, ikt1, ikt2 = consts[c]
                if not ikn > 0:
                    continue
                vn, v1, v2 = (float(Jr @ u) for Jr in J)
                ln, lt1, lt2 = lam[c]
                ln_new = max(0.0, ln + (-vn + bias - gamma * ln) * ikn)
                lim = mu * ln_new
                lt1_new = min(max(lt1 - v1 * ikt1, -lim), lim) if ikt1 > 0 else lt1
                lt2_new = min(max(lt2 - v2 * ikt2, -lim), lim) if ikt2 > 0 else lt2
                u = u + minv * (J[0] * (ln_new - ln) + J[1] * (lt1_new - lt1) + J[2] * (lt2_new - lt2))
                lam[c] = np.array([ln_new, lt1_new, lt2_new])
        for f in range(len(free)):
            v, w = u[nb + 6 * f:nb + 6 * f + 3], Rf[f] @ u[nb + 6 * f + 3:nb + 6 * f + 6]
            free[f][7:10], free[f][10:13] = v, w
            free[f][0:3] = free[f][0:3] + h * v
            qt = free[f][3:7] + 0.5 * h * qmul(np.array([w[0], w[1], w[2], 0.0]), free[f][3:7])
            free[f][3:7] = qt / np.linalg.norm(qt)
        contact_cb.ncontacts.append(len(contacts))
        return u[:nb].copy()

    contact_cb.ncontacts = []
    return contact_cb


def check_push_scene(which="heijn", verbose=True, K=48, steps=(0, 3, 6, 9)):
    """heijn_push with its two static obstacles (BASELINE C4 geometry) or boxer_push (C3: planar base + wheels, 2 substeps), the robot
    really pushing the block: lock-step against the oracle (its state re-injected before every compared step), a few rollouts of
    random commands"""
    import ctypes
    from oracle import oracle as orc
    from scenes import boxer_setup, push_setup
    T = 10
    if which == "pick":
        from test_gpu_sizes import _pick_scene             # panda + gripper (9 joints, tree), block on the table; fingers closing
        T = 30
        sc, p, s0 = _pick_scene(K, T)
        for s_ in range(sc.model.nshapes):                 # per-rollout randomisation off (the restatement has no Philox)
            sc.model.shape_fric_pct[s_] = 0.0
            for c_ in range(3):
                sc.model.shape_size_sigma[s_][c_] = 0.0
        for f_ in range(sc.model.nfree):
            sc.model.free_mass_pct[f_] = 0.0
        a = np.random.default_rng(5).uniform(-0.2, 0.2, (T, sc.nu, K)).astype(np.float32)
        a[:, 7:9] = -0.15 + 0.05 * a[:, 7:9]
    elif which == "heijn":
        sc, p, s0 = push_setup(K=K, T=T, noise=False, block_pos=(0.62, 1.5, 0.1))
        a = np.random.default_rng(3).uniform(-0.6, 0.6, (T, 3, K)).astype(np.float32)
        a[:, 0] = 0.5 + 0.1 * a[:, 0]
    else:
        sc, p, s0 = boxer_setup(K=K, T=T, noise=False)
        rng = np.random.default_rng(0)
        a = np.stack([rng.uniform(0.3, 1.2, (T, K)), rng.uniform(-1.0, 1.0, (T, K))], axis=1).astype(np.float32)
    m = sc.model
    nb, nd2 = m.nb, 2 * sc.ndof
    NS = orc.lib().oracle_state_size(ctypes.byref(m))
    state = np.zeros((NS, K), np.float32)
    state[:nd2] = s0[:, None]
    free_actor = m.free_actor[0]
    state[nd2:nd2 + 13] = sc.root_state0[free_actor][:, None]
    worst_x = worst_v = 0.0
    most = 0
    p1 = _one_step(p)
    for t in range(T):
        before = state.copy()
        state, _ = orc.rollout(m, p, None, a, t, 1, state=state, root0=sc.root_state0, want_obs=False, use_double=True)
        if t not in steps:
            continue
        for k in range(0, K, 6):
            free = [before[nd2:nd2 + 13, k].astype(float)]
            cb = make_contact_phase(m, p, sc.root_state0, free)
            q, qd = rollout(m, p1, before[:nd2, k].astype(float), a[t:t + 1, :, k].astype(float), contact_cb=cb)
            most = max(most, max(cb.ncontacts))
            mine = np.concatenate([q, qd, free[0]])
            refk = state[:nd2 + 13, k].astype(float)
            pos = list(range(nb)) + list(range(nd2, nd2 + 7)); velr = list(range(nb, nd2)) + list(range(nd2 + 7, nd2 + 13))
            worst_x = max(worst_x, np.abs(mine[pos] - refk[pos]).max()); worst_v = max(worst_v, np.abs(mine[velr] - refk[velr]).max())
    if verbose:
        print(f"{'panda_pick' if which == 'pick' else which + '_push'}, lock-step on steps {steps}, {len(range(0, K, 6))} rollouts each: max |position / quaternion difference| = {worst_x:.2e}, "
              f"max |velocity difference| = {worst_v:.2e}; up to {most} contacts per substep")
    assert most >= (4 if which == "pick" else 8), "the robot must have been pushing"
    assert worst_x < 2e-6 and worst_v < 2e-5, (worst_x, worst_v)
    return worst_x, worst_v


def _one_step(p):
    import copy
    p1 = copy.copy(p)
    p1.T = 1
    return p1


if __name__ == "__main__":
    check()
    check_free_box()
    check_push_scene("heijn")
    check_push_scene("boxer", steps=(0, 4, 7, 9))
    check_push_scene("pick", K=12, steps=(0, 10, 20, 29))
