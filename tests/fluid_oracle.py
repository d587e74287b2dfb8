"""TEST INFRASTRUCTURE -- the cold relativistic fluid of WarpXFluidContainer restated in numpy, stage by stage, in the
reference's expression order (paths relative to Source/ of ECP-WarpX/WarpX; numpy rounds every operation, as the
reference's CPU build does):

    gather_push      <- WarpXFluidContainer::GatherAndPush        Fluids/WarpXFluidContainer.cpp:967-1238
    advect           <- WarpXFluidContainer::AdvectivePush_Muscl  :421-893, leaves Fluids/MusclHancockUtils.H
    deposit_current  <- WarpXFluidContainer::DepositCurrent       :1276-1398
    deposit_charge   <- WarpXFluidContainer::DepositCharge        :1240-1273

A fluid state is four numpy arrays [k, j, i] (N, NUx, NUy, NUz) over one all-nodal box with 2 guard nodes, described
by an abi.pic_fab.  FluidRun drives the deck loop: the fluid stages in the position of WarpX::PushParticlesandDeposit
(Evolve/WarpXEvolve.cpp:1171-1178) and the field solve and guard-cell exchanges of the C++ oracle's stage functions
(oracle/pic_oracle.cpp), on one box."""
import ctypes as C
import math

import numpy as np

from warpx_b200 import abi, engine

CL = 299792458.0


def _where_min(a, b):          # std::min
    return np.where(b < a, b, a)


def _where_max(a, b):          # std::max
    return np.where(a < b, b, a)


def minmod3(a, b, c):
    pos = (a > 0.0) & (b > 0.0) & (c > 0.0)
    neg = (a < 0.0) & (b < 0.0) & (c < 0.0)
    return np.where(pos, _where_min(a, _where_min(b, c)), np.where(neg, _where_max(a, _where_max(b, c)), 0.0))


def ave(a, b):
    return np.where(a * b > 0.0, minmod3((a + b) / 2.0, 2.0 * a, 2.0 * b), 0.0)


def _primitive(N, NU):
    with np.errstate(divide="ignore", invalid="ignore"):
        return [np.where(N > 0.0, v / N, 0.0) for v in NU]


AX = (2, 1, 0)      # direction d -> numpy axis


def advect(state, desc, dx, dt, counters=None):
    """AdvectivePush_Muscl on the valid nodes of `state` (guards filled); returns the new state (valid nodes updated,
    guards copied).  counters: a dict that receives the number of valid nodes with N <= 0 ("zero_edges") and of
    directions the positivity limiter reset at valid nodes ("limited")."""
    N, NU = state[0], state[1:]
    ng = [desc.ng[d] for d in range(3)]
    nv = [desc.hi[d] - desc.lo[d] + 1 - 2 * ng[d] for d in range(3)]
    assert min(ng) >= 2
    U = _primitive(N, NU)
    c_sq = CL * CL
    h = [0.5 * (dt / dx[d]) for d in range(3)]
    dtdx = [(dt / dx[d]) for d in range(3)]
    # prediction over the valid nodes grown by one: region P (start ng-1, length nv+2 per direction)
    P = tuple(slice(ng[a] - 1, ng[a] - 1 + nv[a] + 2) for a in (2, 1, 0))
    Pn = [nv[a] + 2 for a in (2, 1, 0)]       # numpy-axis lengths

    def nb(a, d, s):
        """a over P shifted by s along direction d."""
        sl = list(P)
        ax = AX[d]
        sl[ax] = slice(P[ax].start + s, P[ax].stop + s)
        return a[tuple(sl)]

    n0 = N[P]
    u = [v[P] for v in U]
    pos = n0 > 0.0
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        gamma = np.sqrt(1.0 + (u[0] * u[0] + u[1] * u[1] + u[2] * u[2]) / (c_sq))
        inv = 1.0 / (c_sq * gamma * gamma * gamma)
        dU = [[None] * 4 for _ in range(3)]
        JdU = [[None] * 4 for _ in range(3)]
        for d in range(3):
            dU[d][0] = ave(n0 - nb(N, d, -1), nb(N, d, 1) - n0)
            for c in range(3):
                dU[d][1 + c] = ave(u[c] - nb(U[c], d, -1), nb(U[c], d, 1) - u[c])
            V = u[d] / gamma
            J0 = [n0 * (1 / gamma) * (1 - V * V / c_sq) if c == d else -n0 * u[c] * u[d] * inv for c in range(3)]
            JdU[d][0] = V * dU[d][0] + J0[0] * dU[d][1] + J0[1] * dU[d][2] + J0[2] * dU[d][3]
            for c in range(1, 4):
                JdU[d][c] = V * dU[d][c]
        base = [n0, u[0], u[1], u[2]]
        hi = [[None] * 4 for _ in range(3)]
        lo = [[None] * 4 for _ in range(3)]
        for c in range(4):
            ut = base[c] - h[0] * JdU[0][c] - h[1] * JdU[1][c] - h[2] * JdU[2][c]
            for d in range(3):
                hi[d][c] = ut + dU[d][c] / 2.0
                lo[d][c] = ut - dU[d][c] / 2.0
    nlim = 0
    for d in range(3):
        ax = AX[d]
        p = np.arange(Pn[ax]).reshape([-1 if a == ax else 1 for a in range(3)])
        have_hi = p <= Pn[ax] - 2               # node index <= vhi
        have_lo = p >= 1                         # node index >= vlo
        reset_hi = pos & have_hi & ((hi[d][0] < 0.0) | (have_lo & (lo[d][0] < 0.0)))
        reset_lo = pos & have_lo & ((lo[d][0] < 0.0) | (have_hi & (hi[d][0] < 0.0)))
        inner = tuple(slice(1, 1 + nv[a]) for a in (2, 1, 0))
        nlim += int(np.count_nonzero((reset_hi | reset_lo)[inner]))
        for c in range(4):
            hi[d][c] = np.where(pos, np.where(reset_hi, base[c], hi[d][c]), 0.0)
            lo[d][c] = np.where(pos, np.where(reset_lo, base[c], lo[d][c]), 0.0)
    if counters is not None:
        inner = tuple(slice(1, 1 + nv[a]) for a in (2, 1, 0))
        counters["zero_edges"] = counters.get("zero_edges", 0) + int(np.count_nonzero(~pos[inner]))
        counters["limited"] = counters.get("limited", 0) + nlim

    def vcalc(e, d):
        g = np.sqrt(1.0 + (e[1] * e[1] + e[2] * e[2] + e[3] * e[3]) / (CL * CL))
        return e[1 + d] / g

    def flux(m, p, k, vm, vp):
        cc = _where_max(np.abs(vm), np.abs(vp))
        if k == 0:
            return 0.5 * (vm * m[0] + vp * p[0]) - (0.5 * cc) * (p[0] - m[0])
        return 0.5 * (vm * m[0] * m[k] + vp * p[0] * p[k]) - (0.5 * cc) * (p[0] * p[k] - m[0] * m[k])

    def sub(e, d, s):
        """edge arrays over P -> valid nodes shifted by s along d."""
        out = []
        for a_ in e:
            sl = [slice(1, 1 + nv[a]) for a in (2, 1, 0)]
            sl[AX[d]] = slice(1 + s, 1 + s + nv[d])
            out.append(a_[tuple(sl)])
        return out

    dF = [[None] * 4 for _ in range(3)]
    for d in range(3):
        Hs, Ls = sub(hi[d], d, 0), sub(lo[d], d, 0)
        R, Lft = sub(lo[d], d, 1), sub(hi[d], d, -1)
        vm_i, vp_i = vcalc(Hs, d), vcalc(R, d)
        vm_l, vp_l = vcalc(Lft, d), vcalc(Ls, d)
        for c in range(4):
            dF[d][c] = flux(Hs, R, c, vm_i, vp_i) - flux(Lft, Ls, c, vm_l, vp_l)
    out = [a.copy() for a in state]
    V = desc.valid_slices()
    for c in range(4):
        out[c][V] = state[c][V] - dtdx[0] * dF[0][c] - dtdx[1] * dF[1][c] - dtdx[2] * dF[2][c]
    return out


def interp_to_node(F, fdesc, udesc):
    """ablastr::coarsen::sample::Interp (cr = 1) of component F (descriptor fdesc) at the valid nodes of udesc."""
    sf = [fdesc.stag[d] for d in range(3)]
    npt = [2 - sf[d] for d in range(3)]
    vlo = [udesc.lo[d] + udesc.ng[d] for d in range(3)]
    nv = [udesc.hi[d] - udesc.lo[d] + 1 - 2 * udesc.ng[d] for d in range(3)]
    w = (1.0 / npt[0]) * (1.0 / npt[1]) * (1.0 / npt[2])
    c = np.zeros((nv[2], nv[1], nv[0]))
    for kr in range(npt[2]):
        for jr in range(npt[1]):
            for ir in range(npt[0]):
                s = [vlo[d] - (1 - sf[d]) + (ir, jr, kr)[d] - fdesc.lo[d] for d in range(3)]
                c = c + w * F[s[2]:s[2] + nv[2], s[1]:s[1] + nv[1], s[0]:s[0] + nv[0]]
    return c


def push_hc(ux, uy, uz, Ex, Ey, Ez, Bx, By, Bz, q, m, dt):
    """UpdateMomentumHigueraCary (Particles/Pusher/UpdateMomentumHigueraCary.H:21-64)."""
    qmt = 0.5 * q * dt / m
    invclight = 1.0 / CL
    invclightsq = 1.0 / (CL * CL)
    umx, umy, umz = ux + qmt * Ex, uy + qmt * Ey, uz + qmt * Ez
    gamma = 1.0 + (umx * umx + umy * umy + umz * umz) * invclightsq
    betax, betay, betaz = qmt * Bx, qmt * By, qmt * Bz
    betam = betax * betax + betay * betay + betaz * betaz
    sigma = gamma - betam
    ust = (umx * betax + umy * betay + umz * betaz) * invclight
    gamma = 1.0 / np.sqrt(0.5 * (sigma + np.sqrt(sigma * sigma + 4.0 * (betam + ust * ust))))
    tx, ty, tz = gamma * betax, gamma * betay, gamma * betaz
    s = 1.0 / (1.0 + (tx * tx + ty * ty + tz * tz))
    umt = umx * tx + umy * ty + umz * tz
    upx = s * (umx + umt * tx + umy * tz - umz * ty)
    upy = s * (umy + umt * ty + umz * tx - umx * tz)
    upz = s * (umz + umt * tz + umx * ty - umy * tx)
    return (upx + qmt * Ex + upy * tz - upz * ty, upy + qmt * Ey + upz * tx - upx * tz,
            upz + qmt * Ez + upx * ty - upy * tx)


def gather_push(state, desc, E, B, q, m, dt):
    """GatherAndPush in place on the valid nodes with N > 0.  E, B: lists of (descriptor, array)."""
    V = desc.valid_slices()
    N = state[0][V]
    F = [interp_to_node(a, d, desc) for d, a in list(E) + list(B)]
    pos = N > 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        u = [state[1 + c][V] / N for c in range(3)]
        ux, uy, uz = push_hc(*u, *F, q, m, dt)
    for c, v in enumerate((ux, uy, uz)):
        state[1 + c][V] = np.where(pos, N * v, state[1 + c][V])


def _owned(desc):
    """numpy slices of the owned nodes [box_lo, box_hi] of an all-nodal valid box."""
    return tuple(slice(desc.ng[d], desc.hi[d] - desc.lo[d] + 1 - desc.ng[d] - 1) for d in (2, 1, 0))


def deposit_current(state, desc, J, q):
    """DepositCurrent: J (list of (descriptor, array), Yee) += the interpolated q NU / gamma at the owned points."""
    N, NU = state[0], state[1:]
    inv_clight_sq = 1.0 / CL / CL
    with np.errstate(divide="ignore", invalid="ignore"):
        U = [np.where(N > 0.0, v / N, 0.0) for v in NU]
        gamma = np.where(N > 0.0, np.sqrt(1.0 + (U[0] * U[0] + U[1] * U[1] + U[2] * U[2]) * inv_clight_sq), 1.0)
    nown = [desc.hi[d] - desc.lo[d] + 1 - 2 * desc.ng[d] - 1 for d in range(3)]
    for c, (jd, ja) in enumerate(J):
        tmp = q * (NU[c] / gamma)
        npt = [2 - jd.stag[d] for d in range(3)]
        w = (1.0 / npt[0]) * (1.0 / npt[1]) * (1.0 / npt[2])
        acc = np.zeros((nown[2], nown[1], nown[0]))
        for kr in range(npt[2]):
            for jr in range(npt[1]):
                for ir in range(npt[0]):
                    s = [desc.ng[d] + (ir, jr, kr)[d] for d in range(3)]
                    acc = acc + w * tmp[s[2]:s[2] + nown[2], s[1]:s[1] + nown[1], s[0]:s[0] + nown[0]]
        o = [jd.ng[d] for d in range(3)]
        ja[o[2]:o[2] + nown[2], o[1]:o[1] + nown[1], o[0]:o[0] + nown[0]] += acc


def deposit_charge(state, desc, rdesc, rho, q):
    """DepositCharge: rho (nodal, same box) += q N at the owned nodes."""
    n = [desc.hi[d] - desc.lo[d] + 1 - 2 * desc.ng[d] - 1 for d in range(3)]
    a = state[0][_owned(desc)]
    o = [rdesc.ng[d] for d in range(3)]
    rho[o[2]:o[2] + n[2], o[1]:o[1] + n[1], o[0]:o[0] + n[0]] += q * a


def initial_state(desc, prob_lo, dx, box_lo, density, momentum):
    """InitData (:166-254), lab frame: x = prob_lo + i dx over the valid nodes, N = n, NU = n u c; guards zero."""
    nv = [desc.hi[d] - desc.lo[d] + 1 - 2 * desc.ng[d] for d in range(3)]
    coords = [prob_lo[d] + np.arange(box_lo[d], box_lo[d] + nv[d]) * dx[d] for d in range(3)]
    Z, Y, X = np.meshgrid(coords[2], coords[1], coords[0], indexing="ij")
    n = np.broadcast_to(np.asarray(density(X, Y, Z), dtype=np.float64), X.shape)
    u = [np.broadcast_to(np.asarray(v, dtype=np.float64), X.shape) for v in momentum(X, Y, Z)]
    state = [np.zeros(desc.shape) for _ in range(4)]
    V = desc.valid_slices()
    state[0][V] = n
    for c in range(3):
        state[1 + c][V] = n * (u[c] * CL)
    return state


class FluidRun:
    """Fluids (and no particles) on one periodic box through WarpX::Evolve: fields from the C++ oracle's stage
    functions, the fluid stages from this module."""

    def __init__(self, orc, n_cell, prob_lo, prob_hi, cfl=1.0, box_lo=(0, 0, 0)):
        self.L = orc.lib()
        self.n_cell, self.prob_lo, self.prob_hi = tuple(n_cell), tuple(prob_lo), tuple(prob_hi)
        self.dx = [(prob_hi[d] - prob_lo[d]) / n_cell[d] for d in range(3)]
        self.dt = cfl * engine.max_dt(abi.SOLVER_YEE, self.dx)
        g = engine.guard_cells(1, self.dt, self.dx)
        self.g = g
        self.box_lo = (0, 0, 0)
        self.box_hi = tuple(n - 1 for n in n_cell)
        self.geom = abi.make_geom(n_cell, prob_lo, prob_hi)
        self.st = engine.stencil_coefficients(abi.SOLVER_YEE, self.dx)
        self.fabs = [orc.HostFab(self.box_lo, self.box_hi, g["ng_EB"] if c < 6 else g["ng_J"], abi.YEE_STAG[c])
                     for c in range(9)]
        self.orc = orc
        self.fluids = []
        self.is_synchronized = True
        self.counters = {}

    def add_fluid(self, q, m, density, momentum):
        desc = abi.make_fab(None, self.box_lo, self.box_hi, (2, 2, 2), (1, 1, 1))
        st = initial_state(desc, self.prob_lo, self.dx, self.box_lo, density, momentum)
        self.fluids.append(dict(q=q, m=m, desc=desc, state=st))

    def _fill(self, comps, ng):
        arr = self.orc.fab_array([self.fabs[c] for c in comps])
        for n in range(len(comps)):
            self.L.orc_fill_boundary(C.byref(arr[n]), 1, abi.int3(ng), C.byref(self.geom))

    def fill_fluid(self, fl):
        for a in fl["state"]:
            d = abi.make_fab(a.ctypes.data, self.box_lo, self.box_hi, (2, 2, 2), (1, 1, 1))
            self.L.orc_fill_boundary(C.byref(d), 1, abi.int3((2, 2, 2)), C.byref(self.geom))

    def step(self, last):
        g = self.g
        self._fill(range(6), g["ng_EB"] if self.is_synchronized else g["ng_FG"])
        self.is_synchronized = False
        for c in range(6, 9):
            self.fabs[c].a[...] = 0.0
        E = [(self.fabs[c].desc, self.fabs[c].a) for c in range(3)]
        B = [(self.fabs[c].desc, self.fabs[c].a) for c in range(3, 6)]
        J = [(self.fabs[c].desc, self.fabs[c].a) for c in range(6, 9)]
        for fl in self.fluids:
            gather_push(fl["state"], fl["desc"], E, B, fl["q"], fl["m"], self.dt)
            self.fill_fluid(fl)
            fl["state"] = advect(fl["state"], fl["desc"], self.dx, self.dt, self.counters)
            deposit_current(fl["state"], fl["desc"], J, fl["q"])
        arr = self.orc.fab_array(self.fabs[6:9])
        for n in range(3):
            self.L.orc_sum_boundary(C.byref(arr[n]), 1, abi.int3(g["ng_depos_J"]), abi.int3(g["ng_J"]), C.byref(self.geom))
        Ep, Bp, Jp = (self.orc.fab_array(self.fabs[c:c + 3]) for c in (0, 3, 6))
        self.L.orc_evolve_b(Bp, Ep, C.byref(self.st), 0.5 * self.dt)
        self._fill(range(3, 6), g["ng_FS"])
        self.L.orc_evolve_e(Ep, Bp, Jp, C.byref(self.st), self.dt)
        self._fill(range(3), g["ng_FS"])
        self.L.orc_evolve_b(Bp, Ep, C.byref(self.st), 0.5 * self.dt)
        if last:
            self._fill(range(6), g["ng_FG"])
            self.is_synchronized = True

    def evolve(self, nsteps):
        for n in range(nsteps):
            self.step(n == nsteps - 1)

    def checksum_field(self, comp):
        return self.L.orc_checksum_cell_centered(C.byref(self.fabs[comp].desc), abi.int3(self.box_lo),
                                                 abi.int3(self.box_hi))

    def rho(self):
        """The `rho` diagnostic: q N of every fluid at the owned nodes, SumBoundary (RhoFunctor.cpp:47-61)."""
        ng = max(1 + 1 + int(math.ceil(CL * self.dt / self.dx[d])) for d in range(3))
        r = self.orc.HostFab(self.box_lo, self.box_hi, (ng,) * 3, (1, 1, 1))
        for fl in self.fluids:
            deposit_charge(fl["state"], fl["desc"], r.desc, r.a, fl["q"])
        self.L.orc_sum_boundary(C.byref(r.desc), 1, abi.int3((ng,) * 3), abi.int3((ng,) * 3), C.byref(self.geom))
        return r

    def rho_checksum(self):
        r = self.rho()
        return self.L.orc_checksum_cell_centered(C.byref(r.desc), abi.int3(self.box_lo), abi.int3(self.box_hi))

    def field_energy(self):
        """FieldEnergy: (E energy, B energy) over the unique points."""
        e = [self.L.orc_sum_squares_unique(C.byref(self.fabs[c].desc), 1, C.byref(self.geom)) for c in range(6)]
        dV = self.dx[0] * self.dx[1] * self.dx[2]
        return 0.5 * sum(e[:3]) * engine.EP0 * dV, 0.5 * sum(e[3:]) / engine.MU0 * dV
