"""TEST INFRASTRUCTURE -- seeded particle sets for the collision stage and a runner of pic_collide_pairwise_coulomb that
works with the device library (CUDA tensors) and with the host build of tests/host_harness (CPU tensors)."""
import ctypes as C

import numpy as np

from warpx_b200 import abi, workloads

ME, QE = workloads.M_E, workloads.Q_E
GEOM = dict(n_cell=(6, 5, 4), prob_lo=(0.0, -1.0e-6, 2.0e-6), prob_hi=(3.0e-6, 1.5e-6, 4.0e-6),
            box_lo=(0, 0, 0), box_hi=(5, 4, 3))


def particle_set(seed, geom, counts, u_th, u_m=(0.0, 0.0, 0.0), weights="equal", id_offset=0, w0=1.0e9):
    """counts: particles per cell of the box (array [k, j, i] or a Poisson mean); positions uniform in each cell,
    momenta N(u_m, u_th^2) c, weights equal or log-uniform over two decades; ids a random permutation; storage order
    random."""
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(geom["box_lo"]), np.asarray(geom["box_hi"])
    shape = tuple(int(v) for v in (hi - lo + 1)[::-1])
    cnt = rng.poisson(counts, size=shape) if np.ndim(counts) == 0 else np.asarray(counts).reshape(shape)
    dx = [(geom["prob_hi"][d] - geom["prob_lo"][d]) / geom["n_cell"][d] for d in range(3)]
    K, J, I = np.meshgrid(*[np.arange(lo[d], hi[d] + 1) for d in (2, 1, 0)], indexing="ij")
    cells = [np.repeat(a.ravel(), cnt.ravel()) for a in (I, J, K)]
    n = len(cells[0])
    pos = [geom["prob_lo"][d] + (cells[d] + rng.uniform(0.02, 0.98, n)) * dx[d] for d in range(3)]
    u = [(u_m[d] + u_th[d] * rng.standard_normal(n)) * workloads.C for d in range(3)]
    w = np.full(n, w0) if weights == "equal" else w0 * 10.0 ** rng.uniform(-1.0, 1.0, n)
    ids = rng.permutation(n).astype(np.int64) + id_offset
    order = rng.permutation(n)
    sp = dict(x=pos[0], y=pos[1], z=pos[2], w=w, ux=u[0], uy=u[1], uz=u[2], id=ids)
    return {k: np.ascontiguousarray(v[order]) for k, v in sp.items()}


def make_geom(geom):
    return abi.make_geom(geom["n_cell"], geom["prob_lo"], geom["prob_hi"])


class DeviceSpecies:
    """Two SoA buffers + ids + bins of one particle set on the library's device (or the host build's CPU tensors)."""
    NAMES = ("x", "y", "z", "w", "ux", "uy", "uz")

    def __init__(self, L, t, dev, sp, geom, tile=(8, 8, 8), stream=None):
        self.L, self.t, self.n = L, t, len(sp["x"])
        cap = max(self.n, 1)
        self.buf = [t.zeros((7, cap), dtype=t.float64, device=dev) for _ in range(2)]
        self.ids = [t.zeros(cap, dtype=t.int64, device=dev) for _ in range(2)]
        for k, name in enumerate(self.NAMES):
            self.buf[0][k, :self.n] = t.from_numpy(sp[name].copy())
        self.ids[0][:self.n] = t.from_numpy(sp["id"].copy())
        self.bins = abi.pic_bins()
        for d in range(3):
            self.bins.box_lo[d], self.bins.box_hi[d], self.bins.tile[d] = geom["box_lo"][d], geom["box_hi"][d], tile[d]
        nb = L.pic_bins_count(abi.int3(geom["box_lo"]), abi.int3(geom["box_hi"]), abi.int3(tile))
        self.cell_start = t.zeros(nb + 1, dtype=t.int32, device=dev)
        self.work = t.zeros(L.pic_sort_workspace_bytes(cap, nb), dtype=t.uint8, device=dev)
        self.bins.cell_start = self.cell_start.data_ptr()
        self.g = make_geom(geom)
        self.stream = stream
        self.src = None
        self.cur = 0

    def soa(self, b):
        s = abi.pic_soa()
        for k, name in enumerate(self.NAMES):
            setattr(s, name, self.buf[b][k].data_ptr())
        s.idcpu, s.np = self.ids[b].data_ptr(), self.n
        return s

    def sort(self, pending):
        """cell sort: pending=True leaves the particles in place and keeps the permutation src, else moves them"""
        src = C.c_void_p()
        assert self.L.pic_sort_index_by_cell(C.byref(self.soa(0)), C.byref(self.g), C.byref(self.bins),
                                             self.work.data_ptr(), C.byref(src), self.stream) == 0
        self.bins.np_binned = self.n
        if pending:
            self.src, self.cur = src.value, 0
        else:
            assert self.L.pic_sort_apply_permutation(C.byref(self.soa(0)), C.byref(self.soa(1)), src, self.stream) == 0
            self.src, self.cur = None, 1

    def numpy(self):
        """every array of the current buffer, and the ids, in storage order"""
        out = {name: self.buf[self.cur][k, :self.n].cpu().numpy().copy() for k, name in enumerate(self.NAMES)}
        out["id"] = self.ids[self.cur][:self.n].cpu().numpy().copy()
        return out


def collision_spec(coll):
    c = abi.pic_coulomb_collision()
    for k in ("q1", "m1", "q2", "m2", "coulomb_log", "seed", "collision_index", "same_species"):
        setattr(c, k, coll[k])
    return c


def run_stage(L, t, dev, sp1, sp2, coll, geom, dt, step, pending=True, stream=None, sync=lambda: None, scratch=True):
    """pic_collide_pairwise_coulomb on fresh copies of sp1 (and sp2): returns (species 1, species 2 or None, status),
    each species as dict of arrays by storage order of the buffer the stage worked on, with the ids."""
    d1 = DeviceSpecies(L, t, dev, sp1, geom, stream=stream)
    d1.sort(pending)
    d2 = None
    if not coll["same_species"]:
        d2 = DeviceSpecies(L, t, dev, sp2, geom, stream=stream)
        d2.sort(pending)
    status = t.zeros(1, dtype=t.int32, device=dev)
    o = d2 if d2 is not None else d1
    rc = L.pic_collide_pairwise_coulomb(C.byref(collision_spec(coll)), C.byref(d1.soa(d1.cur)), C.byref(d1.bins), d1.src,
                                        C.byref(o.soa(o.cur)), C.byref(o.bins), o.src, C.byref(d1.g), dt, step,
                                        L.pic_sort_scratch(d1.work.data_ptr(), d1.n) if scratch else None,
                                        L.pic_sort_scratch(o.work.data_ptr(), o.n) if scratch else None,
                                        status.data_ptr(), stream)
    assert rc == 0, L.pic_last_error()
    sync()
    return d1.numpy(), (d2.numpy() if d2 is not None else None), int(status.cpu()[0])


def by_id(sp):
    o = np.argsort(sp["id"], kind="stable")
    return {k: v[o] for k, v in sp.items() if isinstance(v, np.ndarray)}


def ee_spec(L=-1.0, seed=7, cidx=0):
    return dict(q1=-QE, m1=ME, q2=-QE, m2=ME, coulomb_log=L, seed=seed, collision_index=cidx, same_species=1)


def ei_spec(L=-1.0, seed=7, cidx=1, mi=5 * ME):
    return dict(q1=-QE, m1=ME, q2=QE, m2=mi, coulomb_log=L, seed=seed, collision_index=cidx, same_species=0)


def reference_cases():
    """The cases of tests/golden/collision_reference.npz (make_collision_reference.py): name -> (sp1, sp2 or None,
    coll, geom, dt, step, u1, u2 or None), u = what the reference's headers computed, (3, np) in storage order."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "collision_reference.npz"))
    out = {}
    for name in sorted({k.split("/")[0] for k in z.files}):
        p = name + "/"
        sp1 = {k[len(p) + 4:]: z[k] for k in z.files if k.startswith(p + "sp1_")}
        sp2 = {k[len(p) + 4:]: z[k] for k in z.files if k.startswith(p + "sp2_")} or None
        c, i, g = z[p + "coll"], z[p + "ints"], z[p + "geom"]
        coll = dict(q1=c[0], m1=c[1], q2=c[2], m2=c[3], coulomb_log=c[4], seed=int(i[0]), collision_index=int(i[1]),
                    same_species=int(i[2]))
        geom = dict(n_cell=tuple(int(v) for v in g[0:3]), prob_lo=tuple(g[3:6]), prob_hi=tuple(g[6:9]),
                    box_lo=tuple(int(v) for v in g[9:12]), box_hi=tuple(int(v) for v in g[12:15]))
        out[name] = (sp1, sp2, coll, geom, float(c[5]), int(c[6]), z[p + "u1"], z[p + "u2"] if sp2 is not None else None)
    return out


def assert_matches_reference(got, sp, u_ref, rtol, geom=GEOM):
    """got: a species after the stage (any storage order, with ids); the reference's u per id, to rtol of the |u| scale
    of the particle's cell (the largest |u| there before or after: the scale of any pair it took part in)"""
    import collision_oracle as co
    ref = dict(sp)
    ref["ux"], ref["uy"], ref["uz"] = u_ref
    got, ref, ini = by_id(got), by_id(ref), by_id(sp)
    mag = np.maximum(np.sqrt(ref["ux"] ** 2 + ref["uy"] ** 2 + ref["uz"] ** 2),
                     np.sqrt(ini["ux"] ** 2 + ini["uy"] ** 2 + ini["uz"] ** 2))
    cell = co.cells_of(ini, geom)
    cmax = np.zeros(int(cell.max()) + 1)
    np.maximum.at(cmax, cell, mag)
    scale = np.maximum(cmax[cell], np.finfo(np.float64).tiny)
    for k in ("ux", "uy", "uz"):
        err = (np.abs(got[k] - ref[k]) / scale).max()
        assert err <= rtol, (k, err)
