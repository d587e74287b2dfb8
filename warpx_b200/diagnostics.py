"""Full diagnostics of a run in the reference's plotfile layout (SURVEY.md section 8f, rank 4).

    write_plotfile(sim, "diags/plt", iteration)   <- FlushFormatPlotfile::WriteToFile
                                                     (Source/Diagnostics/FlushFormats/FlushFormatPlotfile.cpp:61-115)

What WarpX writes for `diag.format = plotfile` and what its regression harness reads back
(Regression/Checksum/checksum.py:62-217 through yt's boxlib frontend):

  <prefix><iteration, 5+ digits>/
      Header                        HyperCLaw-V1.1: variable names, geometry, one box per rank
      Level_0/Cell_H                VisMF header (Version_v1, FlushFormatPlotfile.cpp:91): boxes, FabOnDisk, min / max
      Level_0/Cell_D_<rank>         one FAB per rank: "FAB ((8, (64 11 52 0 1 12 0 1023)),(8, (8 7 6 5 4 3 2 1)))" + box
                                    + ncomp, then ncomp x nx*ny*nz little-endian doubles, Fortran order, valid cells only
      WarpXHeader, warpx_job_info   (FlushFormatPlotfile.cpp:118-340)
      <species>/Header              Version_Two_Dot_Zero_double: 3, the real components "weight momentum_x momentum_y
                                    momentum_z" (:362-366), no integer components, counts per grid
      <species>/Level_0/Particle_H  the boxes again
      <species>/Level_0/DATA_<rank> per particle x y z w px py pz (doubles), momenta in SI units m*u
                                    (particlesConvertUnits, Source/Particles/ParticleIO.H:41-79)

The fields are the cell-centred averages the reference's default `fields_to_plot` go through (CellCenterFunctor ->
ablastr::coarsen::sample::Interp with ratio 1, Source/ablastr/coarsen/sample.H:47-104: along a nodal direction the two
neighbouring nodes are averaged), computed on the device with torch slicing; everything else here is host-side file
writing.  AMReX itself (amrex::WriteMultiLevelPlotfile, ParticleContainer::WritePlotFile; pinned at 62c2a81, not vendored
in the reference tree) defines the byte layout; it is restated here from its documented file format.  yt is not in this
image, so the tests read the files back with tests/plotfile_reader.py, a reader written against the same layout, and
reproduce the reference's stored checksums from them.
"""
import os

import numpy as np

from . import abi

FAB_DESCRIPTOR = "FAB ((8, (64 11 52 0 1 12 0 1023)),(8, (8 7 6 5 4 3 2 1)))"      # IEEE little-endian double


def cell_centered(sim, comp):
    """Component comp (0..8 = Ex..jz) of this rank averaged to the cell centres of its box: torch tensor [nz, ny, nx]
    (ablastr/coarsen/sample.H:69-103 with cr = 1: np = 1 + |stag_src - stag_dst| points, weight 1/np each)."""
    d = sim.fab[comp]
    a = sim.data[comp]
    ng = [d.ng[k] for k in range(3)]
    n = [sim.box_hi[k] - sim.box_lo[k] + 1 for k in range(3)]
    st = abi.YEE_STAG[comp]
    out = None
    # tensor axes are (z, y, x); average over the 2^(number of nodal directions) surrounding nodes
    shifts = [(0, 1) if st[k] else (0,) for k in range(3)]
    count = 0
    for sz in shifts[2]:
        for sy in shifts[1]:
            for sx in shifts[0]:
                v = a[ng[2] + sz: ng[2] + sz + n[2], ng[1] + sy: ng[1] + sy + n[1], ng[0] + sx: ng[0] + sx + n[0]]
                out = v.clone() if out is None else out + v
                count += 1
    return out * (1.0 / count)


def _box_str(lo, hi):
    return "((%d,%d,%d) (%d,%d,%d) (0,0,0))" % (lo[0], lo[1], lo[2], hi[0], hi[1], hi[2])


def _gather(sim, values):
    """values (list of python floats / ints of this rank) from every rank, as a [world][len] list (rank order)."""
    if sim.dist is None or sim.world == 1:
        return [list(values)]
    t = sim.torch
    mine = t.tensor(values, dtype=t.float64, device=sim.device)
    parts = [t.empty_like(mine) for _ in range(sim.world)]
    sim.dist.all_gather(parts, mine)
    return [p.cpu().tolist() for p in parts]


def write_plotfile(sim, prefix, iteration=None, fields=("Ex", "Ey", "Ez", "Bx", "By", "Bz", "jx", "jy", "jz"),
                   species=None, file_min_digits=5):
    """Write <prefix><iteration> as the reference's plotfile diagnostic would (every rank its own data files, rank 0 the
    headers).  species: indices to dump (default all).  Returns the directory."""
    from . import parallel
    it = sim.istep if iteration is None else int(iteration)
    root = "%s%0*d" % (prefix, file_min_digits, it)
    lev = os.path.join(root, "Level_0")
    rank, world = sim.rank, sim.world
    if rank == 0:
        os.makedirs(lev, exist_ok=True)
    if sim.dist is not None and world > 1:
        sim.dist.barrier()
    comps = [abi.COMP_NAMES.index(f) for f in fields]
    # ---- fields: one FAB per rank ----
    cc = [cell_centered(sim, c).cpu().numpy() for c in comps]
    with open(os.path.join(lev, "Cell_D_%05d" % rank), "wb") as f:
        f.write(("%s%s %d\n" % (FAB_DESCRIPTOR, _box_str(sim.box_lo, sim.box_hi), len(comps))).encode())
        for a in cc:
            f.write(np.ascontiguousarray(a, dtype="<f8").tobytes())      # [z][y][x] C order == Fortran order (x fastest)
    mins = _gather(sim, [float(a.min()) for a in cc])
    maxs = _gather(sim, [float(a.max()) for a in cc])
    boxes = [parallel.Decomposition(sim.n_cell, sim.dec.nb, r) for r in range(world)]
    dx = sim.dx
    time = getattr(sim, "time", 0.0)
    if rank == 0:
        with open(os.path.join(root, "Header"), "w") as f:
            f.write("HyperCLaw-V1.1\n%d\n" % len(fields))
            for name in fields:
                f.write(name + "\n")
            f.write("3\n%.17g\n0\n" % time)
            f.write(" ".join("%.17g" % v for v in sim.prob_lo) + " \n")
            f.write(" ".join("%.17g" % v for v in sim.prob_hi) + " \n")
            f.write("\n")                                                  # refinement ratios: none on one level
            f.write(_box_str((0, 0, 0), tuple(v - 1 for v in sim.n_cell)) + " \n")
            f.write("%d \n" % it)
            f.write(" ".join("%.17g" % v for v in dx) + " \n")
            f.write("0\n0\n")                                              # Cartesian, boundary width
            f.write("0 %d %.17g\n%d\n" % (world, time, it))
            for b in boxes:
                for d in range(3):
                    f.write("%.17g %.17g\n" % (sim.prob_lo[d] + b.box_lo[d] * dx[d], sim.prob_lo[d] + (b.box_hi[d] + 1) * dx[d]))
            f.write("Level_0/Cell\n")
        with open(os.path.join(lev, "Cell_H"), "w") as f:
            f.write("1\n1\n%d\n0\n" % len(comps))                          # Version_v1, NFiles, ncomp, ngrow
            f.write("(%d 0\n" % world)
            for b in boxes:
                f.write(_box_str(b.box_lo, b.box_hi) + "\n")
            f.write(")\n%d\n" % world)
            for r in range(world):
                f.write("FabOnDisk: Cell_D_%05d 0\n" % r)
            f.write("\n")
            for table in (mins, maxs):
                f.write("%d,%d\n" % (world, len(comps)))
                for r in range(world):
                    f.write(",".join("%.17g" % v for v in table[r]) + ",\n")
                f.write("\n")
        with open(os.path.join(root, "WarpXHeader"), "w") as f:            # FlushFormatPlotfile::WriteWarpXHeader (:243-340)
            f.write("Checkpoint version: 1\n1\n%d \n%.17g \n%.17g \n%.17g \n" % (it, sim.dt, time, time - sim.dt))
            f.write(" ".join("%.17g" % v for v in sim.prob_lo) + " \n" + " ".join("%.17g" % v for v in sim.prob_hi) + " \n")
        with open(os.path.join(root, "warpx_job_info"), "w") as f:
            f.write("=" * 78 + "\n warpx_b200 job information\n" + "=" * 78 + "\n")
            f.write("number of ranks (one per GPU): %d\nparticle shape order: %d\nsolver: %s\n"
                    % (world, sim.nox, "CKC" if sim.solver == abi.SOLVER_CKC else "Yee"))
    # ---- particles ----
    which = range(len(sim.species)) if species is None else species
    for isp in which:
        sp = sim.species[isp]
        sdir = os.path.join(root, sp.name, "Level_0")
        if rank == 0:
            os.makedirs(sdir, exist_ok=True)
        if sim.dist is not None and world > 1:
            sim.dist.barrier()
        P = sim.species_numpy(isp)
        rec = np.empty((len(P["x"]), 7), dtype="<f8")
        for k, name in enumerate(("x", "y", "z", "w")):
            rec[:, k] = P[name]
        for k, name in enumerate(("ux", "uy", "uz")):
            rec[:, 4 + k] = P[name] * sp.m                                 # WarpX_to_SI: momentum = m * u
        with open(os.path.join(sdir, "DATA_%05d" % rank), "wb") as f:
            f.write(rec.tobytes())
        counts = _gather(sim, [float(len(P["x"]))])
        if rank == 0:
            ntot = int(sum(c[0] for c in counts))
            with open(os.path.join(root, sp.name, "Header"), "w") as f:
                f.write("Version_Two_Dot_Zero_double\n3\n4\nweight\nmomentum_x\nmomentum_y\nmomentum_z\n0\n0\n")
                f.write("%d\n%d\n0\n%d\n" % (ntot, ntot + 1, world))
                for r in range(world):
                    f.write("%d %d 0\n" % (r, int(counts[r][0])))
            with open(os.path.join(sdir, "Particle_H"), "w") as f:
                f.write("(%d 0\n" % world)
                for b in boxes:
                    f.write(_box_str(b.box_lo, b.box_hi) + "\n")
                f.write(")\n")
    if sim.dist is not None and world > 1:
        sim.dist.barrier()
    return root


# ------------------------------------------------------------------------------------------------------------
# Checkpoint / restart (FlushFormatCheckpoint::WriteToFile, Source/Diagnostics/FlushFormats/FlushFormatCheckpoint.cpp:
# 32-216; WarpX::InitFromCheckpoint, Source/Diagnostics/WarpXIO.cpp:90-400)
# ------------------------------------------------------------------------------------------------------------
#   <prefix><iteration>/WarpXHeader            "Checkpoint version: 1", levels, istep, nsubsteps, t_new, t_old, dt,
#                                              moving-window position, synchronisation flag, prob_lo, prob_hi, boxes
#   Level_0/{Ex,Ey,Ez,Bx,By,Bz}_fp_H, _D_<r>   the six field arrays WITH their guard cells (VisMF, NoFabHeader_v1: the
#                                              data file holds the raw doubles of the rank's FAB); jx, jy, jz as well when
#                                              the run is synchronised (:93-102: "after restart we need j")
#   <species>/Header, Level_0/DATA_<r>         particle checkpoint: is_checkpoint = 1, the integers (id, cpu) of all
#                                              particles of a grid first, then x y z w ux uy uz per particle
CHK_FIELDS = ("Ex_fp", "Ey_fp", "Ez_fp", "Bx_fp", "By_fp", "Bz_fp", "jx_fp", "jy_fp", "jz_fp")


def write_checkpoint(sim, prefix, iteration=None, file_min_digits=5):
    """Everything a restart needs (periodic or walled domains without a moving window).  Returns the directory."""
    from . import parallel
    if sim.moving_window is not None:
        raise NotImplementedError("checkpoints of moving-window runs (the window position is not restored yet)")
    if getattr(sim, "fluids", None):
        raise NotImplementedError("checkpoints of runs with fluid species (the fluid state is not written yet)")
    it = sim.istep if iteration is None else int(iteration)
    root = "%s%0*d" % (prefix, file_min_digits, it)
    lev = os.path.join(root, "Level_0")
    rank, world = sim.rank, sim.world
    if rank == 0:
        os.makedirs(lev, exist_ok=True)
    if sim.dist is not None and world > 1:
        sim.dist.barrier()
    ncomp = 9 if sim.is_synchronized else 6
    boxes = [parallel.Decomposition(sim.n_cell, sim.dec.nb, r) for r in range(world)]
    for c in range(ncomp):
        d = sim.fab[c]
        with open(os.path.join(lev, "%s_D_%05d" % (CHK_FIELDS[c], rank)), "wb") as f:
            f.write(np.ascontiguousarray(sim.data[c].cpu().numpy(), dtype="<f8").tobytes())
        if rank == 0:
            with open(os.path.join(lev, CHK_FIELDS[c] + "_H"), "w") as f:
                f.write("3\n1\n1\n(%d,%d,%d)\n" % (d.ng[0], d.ng[1], d.ng[2]))     # NoFabHeader_v1, NFiles, 1 comp, ngrow
                f.write("(%d 0\n" % world)
                for b in boxes:      # valid boxes in the index type of the component
                    hi = [b.box_hi[k] + abi.YEE_STAG[c][k] for k in range(3)]
                    f.write("((%d,%d,%d) (%d,%d,%d) (%d,%d,%d))\n" % (tuple(b.box_lo) + tuple(hi) + tuple(abi.YEE_STAG[c])))
                f.write(")\n%d\n" % world)
                for r in range(world):
                    f.write("FabOnDisk: %s_D_%05d 0\n" % (CHK_FIELDS[c], r))
    if rank == 0:
        with open(os.path.join(root, "WarpXHeader"), "w") as f:
            f.write("Checkpoint version: 1\n1\n%d \n1 \n%.17g \n%.17g \n%.17g \n" % (it, sim.time, sim.time - sim.dt, sim.dt))
            f.write("0\n%d\n" % (1 if sim.is_synchronized else 0))              # moving_window_x, is_synchronized
            f.write(" ".join("%.17g" % v for v in sim.prob_lo) + " \n" + " ".join("%.17g" % v for v in sim.prob_hi) + " \n")
            f.write("(%d 0\n" % world)
            for b in boxes:
                f.write(_box_str(b.box_lo, b.box_hi) + "\n")
            f.write(")\n")
            f.write("%d\n" % len(sim.species))
            for sp in sim.species:
                f.write("%s %.17g %.17g\n" % (sp.name, sp.q, sp.m))
    for isp, sp in enumerate(sim.species):
        sdir = os.path.join(root, sp.name, "Level_0")
        if rank == 0:
            os.makedirs(sdir, exist_ok=True)
        if sim.dist is not None and world > 1:
            sim.dist.barrier()
        P = sim.species_numpy(isp)
        n = len(P["x"])
        ints = np.empty((n, 2), dtype="<i4")
        ints[:, 0] = (P["id"] & 0xFFFFFFFF).astype(np.int64).astype("<i4")       # idcpu split like AMReX: id, cpu words
        ints[:, 1] = (P["id"] >> 32).astype("<i4")
        rec = np.empty((n, 7), dtype="<f8")
        for k, name in enumerate(("x", "y", "z", "w", "ux", "uy", "uz")):
            rec[:, k] = P[name]
        with open(os.path.join(sdir, "DATA_%05d" % rank), "wb") as f:
            f.write(ints.tobytes())
            f.write(rec.tobytes())
        counts = _gather(sim, [float(n)])
        if rank == 0:
            ntot = int(sum(c[0] for c in counts))
            with open(os.path.join(root, sp.name, "Header"), "w") as f:
                f.write("Version_Two_Dot_Zero_double\n3\n4\nw\nux\nuy\nuz\n0\n1\n%d\n%d\n0\n%d\n" % (ntot, ntot + 1, world))
                for r in range(world):
                    f.write("%d %d 0\n" % (r, int(counts[r][0])))
    if sim.dist is not None and world > 1:
        sim.dist.barrier()
    return root


def read_checkpoint(sim, root):
    """Load a checkpoint written by write_checkpoint into a freshly constructed Simulation with the same grid, guard
    cells and decomposition and no species yet: fields with guards, the species with their ids, step counter and time."""
    with open(os.path.join(root, "WarpXHeader")) as f:
        h = [ln.strip() for ln in f]
    assert h[0] == "Checkpoint version: 1" and int(h[1]) == 1
    istep, time = int(h[2].split()[0]), float(h[4].split()[0])
    synchronized = int(h[8]) == 1
    if not synchronized:
        raise NotImplementedError("restart from a checkpoint written between the half pushes")
    nbox = int(h[11].split()[0][1:])
    assert nbox == sim.world, "the decomposition of the restart must equal the checkpoint's"
    nsp_line = 11 + nbox + 2
    nsp = int(h[nsp_line])
    species = [h[nsp_line + 1 + k].split() for k in range(nsp)]
    assert not sim.species, "read_checkpoint: add no species before the restart"
    t = sim.torch
    lev = os.path.join(root, "Level_0")
    for c in range(9):
        path = os.path.join(lev, "%s_D_%05d" % (CHK_FIELDS[c], sim.rank))
        a = np.fromfile(path, dtype="<f8")
        assert a.size == sim.data[c].numel(), "guard cells of the restart differ from the checkpoint's (%s)" % CHK_FIELDS[c]
        sim.data[c].copy_(t.from_numpy(a.reshape(tuple(sim.data[c].shape))))
    for name, q, m in species:
        with open(os.path.join(root, name, "Header")) as f:
            ph = [ln.strip() for ln in f]
        assert ph[0] == "Version_Two_Dot_Zero_double" and int(ph[8]) == 1      # is_checkpoint
        ngrids = int(ph[12])
        count = None
        for g in range(ngrids):
            which, cnt, where = (int(v) for v in ph[13 + g].split())
            if which == sim.rank:
                count = cnt
        with open(os.path.join(root, name, "Level_0", "DATA_%05d" % sim.rank), "rb") as f:
            ints = np.frombuffer(f.read(8 * count), dtype="<i4").reshape(count, 2)
            rec = np.frombuffer(f.read(56 * count), dtype="<f8").reshape(count, 7)
        ids = (ints[:, 0].astype(np.int64) & 0xFFFFFFFF) | (ints[:, 1].astype(np.int64) << 32)
        sim.add_species(name, float(q), float(m), *[np.ascontiguousarray(rec[:, k]) for k in range(7)], ids=ids)
    sim.set_step(istep, time)
    sim.is_synchronized = True
    return istep
