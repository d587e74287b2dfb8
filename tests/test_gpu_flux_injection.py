"""GPU tests (-m gpu) of the flux injection (csrc/flux_injection.cu, the `flux_injection` stage of the step driver):
  * the device call against the numpy restatement of tests/flux_oracle.py, on the cases of test_flux_injection_host.py:
    the same counts and ids, positions, momenta and weights within 1e-13 of their scale (device libm may differ from the
    host's in the last bits; a rejection decision that flipped would show as a count or id mismatch);
  * the reference's deck at full size (workloads.flux_injection_3d) through a plotfile, against the restated analysis
    of tests/flux_deck_analysis.py, printing the measured values beside their tolerances;
  * 2 slabs along the normal and 2 x 2 x 1 bricks (threads as ranks over the device NCCL stand-in of
    test_gpu_multirank.py) give the single box's particles bit for bit after the injecting step, ids included, and
    after two more steps the same ids, weights and momenta;
  * on species that hold particles unequally over the bricks, the injected ids equal the single box's (the id counter
    starts at the global particle count on every rank);
  * N steps, a checkpoint and a restart, then N steps equal 2N straight steps bit for bit, with no repeated id; on 2
    slabs the same ids, weights and momenta (the checkpoint carries the id counter);
  * an electromagnetic (Yee, order 3) run with an injector runs, and an injector outside its window adds no launch."""
import ctypes as C
import json

import numpy as np
import pytest

import flux_deck_analysis as fda
import flux_oracle as fo
import plotfile_reader as pr
from warpx_b200 import abi, workloads

pytestmark = pytest.mark.gpu

NAMES = ("x", "y", "z", "w", "ux", "uy", "uz")


@pytest.fixture(scope="module")
def L(cuda):
    from warpx_b200.lib import lib
    L = lib()
    L.pic_set_error_mode(abi.PIC_ERR_RETURN)
    return L


def device_call(L, torch, inj, geom, box, step, t, dt, first_id, index, np0=3, capacity=4000):
    g = abi.make_geom(*geom)
    dev = torch.device("cuda")
    buf = torch.zeros((7, capacity), dtype=torch.float64, device=dev)
    ids = torch.full((capacity,), 7, dtype=torch.int64, device=dev)
    soa = abi.pic_soa()
    for k, name in enumerate(NAMES):
        setattr(soa, name, buf[k].data_ptr())
    soa.idcpu, soa.np = ids.data_ptr(), np0
    nbytes = L.pic_flux_workspace_bytes(C.byref(inj), C.byref(g))
    work = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    used = C.c_uint64(0)
    n = L.pic_add_flux_particles(C.byref(inj), index, C.byref(g), abi.int3(box[0]), abi.int3(box[1]), step, t, dt,
                                 C.byref(soa), capacity, first_id, C.byref(used), work.data_ptr(), nbytes,
                                 torch.cuda.current_stream().cuda_stream)
    assert n >= 0, L.pic_last_error().decode()
    torch.cuda.synchronize()
    got = {name: buf[k, np0:np0 + n].cpu().numpy() for k, name in enumerate(NAMES)}
    got["id"] = ids[np0:np0 + n].cpu().numpy()
    return fo.sort_by_id(got), used.value


def test_device_call_matches_the_restatement(L, cuda):
    import torch
    import test_flux_injection_host as th
    worst = {}
    for name, (kw, box) in sorted(th.CASES.items()):
        inj = abi.make_flux_injector(seed=11, **kw)
        step, dt = 5, 2e-9
        got, used = device_call(L, torch, inj, th.GEOM, box, step, 6 * dt, dt, 1000, 2)
        want, want_used = fo.inject(fo.as_dict(inj), th.GEOM, box[0], box[1], step, 6 * dt, dt, 1000, 2)
        want = fo.sort_by_id(want)
        assert used == want_used
        assert np.array_equal(got["id"], want["id"]), name
        for k in NAMES:
            if len(want[k]) == 0:
                continue
            scale = max(np.abs(want[k]).max(), 1e-300)
            err = float(np.abs(got[k] - want[k]).max() / scale)
            worst[k] = max(worst.get(k, 0.0), err)
            assert err <= 1e-13, (name, k, err)
    print("PARITY", json.dumps(worst))


def build(wl, sim_kw=None):
    from warpx_b200.engine import Simulation
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], solver=abi.SOLVER_NONE, dt=wl["dt"],
                     **(sim_kw or {}))
    for s in wl["species"]:
        sim.add_empty_species(s["name"], s["capacity"], q=s["q"], m=s["m"])
    for s in wl["species"]:
        sim.add_flux_injection(s["name"], abi.make_flux_injector(**s["flux"]))
    return sim


def test_full_size_deck_passes_the_restated_analysis(cuda, tmp_path):
    from warpx_b200 import diagnostics
    wl = workloads.flux_injection_3d()
    sim = build(wl)
    sim.enable_stage_timing()
    sim.Evolve(wl["max_step"])
    stages = sim.stage_ms()
    root = diagnostics.write_plotfile(sim, str(tmp_path / "plt"), wl["max_step"])
    data = {}
    for s in wl["species"]:
        d = pr.read_species(root, s["name"])
        mc = s["m"] * fo.C
        data[s["name"]] = dict(ux=d["momentum_x"] / mc, uy=d["momentum_y"] / mc, uz=d["momentum_z"] / mc, w=d["weight"])
    out = fda.check(wl, data, sim.time)
    print("DECK flux_injection_3d", json.dumps(out))
    print("STAGES", json.dumps({k: stages[k] for k in ("flux_injection", "gather_push", "wrap") if k in stages}))
    for isp in range(len(wl["species"])):
        ids = sim.species_numpy(isp)["id"]
        assert np.unique(ids).size == ids.size


def _small_deck():
    return workloads.flux_injection_3d(n=16, ppc=6.5, max_step=4)


def _union(parts):
    out = []
    for isp in range(len(parts[0])):
        out.append(fo.sort_by_id(fo.concat([p[isp] for p in parts])))
    return out


def _same(a, b):
    for sa, sb in zip(a, b):
        assert len(sa["id"]) == len(sb["id"]) and len(sa["id"]) > 0
        for k in sa:
            assert np.array_equal(np.ascontiguousarray(sa[k]).view(np.int64), np.ascontiguousarray(sb[k]).view(np.int64)), k


@pytest.mark.parametrize("nb", [(1, 1, 2), (2, 2, 1)])
def test_bricks_equal_the_single_box(L, cuda, nb):
    """The step that injects gives the single box's particles bit for bit.  Two more steps push them: every id, weight
    and momentum keeps its bits, the positions agree to 1e-13 of the domain (the push computes positions relative to
    each brick's corner, as test_host_multirank.py allows for pushed particles)."""
    import test_gpu_multirank as mr
    wl = _small_deck()
    nsp = len(wl["species"])
    single = build(wl)
    single.Evolve(1)
    want1 = [single.species_numpy(isp, sort_by_id=True) for isp in range(nsp)]
    single.Evolve(2)
    want3 = [single.species_numpy(isp, sort_by_id=True) for isp in range(nsp)]
    single.close()

    def rank(r, dist):
        sim = build(wl, dict(dist=dist, nb=nb))
        sim.Evolve(1)
        one = [sim.species_numpy(isp) for isp in range(nsp)]
        sim.Evolve(2)
        return one, [sim.species_numpy(isp) for isp in range(nsp)]
    parts = mr.run_ranks(nb[0] * nb[1] * nb[2], rank)
    _same(_union([p[0] for p in parts]), want1)
    got3 = _union([p[1] for p in parts])
    for g, w in zip(got3, want3):
        assert np.array_equal(g["id"], w["id"]) and len(w["id"]) > len(want1[0]["id"])
        for k in ("w", "ux", "uy", "uz"):
            assert np.array_equal(g[k].view(np.int64), w[k].view(np.int64)), k
        for k in ("x", "y", "z"):
            assert np.abs(g[k] - w[k]).max() <= 1e-13 * 8.0, k


class _Gathering:
    """The threads' stand-in for torch.distributed (test_gpu_multirank.DeviceThreadDist) with the all_gather that
    checkpoints use."""

    def __init__(self, dist):
        self.dist = dist

    def __getattr__(self, name):
        return getattr(self.dist, name)

    def all_gather(self, parts, tensor):
        sh = self.dist.shared
        sh.slots[self.dist.rank] = tensor.cpu().clone()
        sh.barrier.wait()
        for r, part in enumerate(parts):
            part.copy_(sh.slots[r])
        sh.barrier.wait()


def _seeded(wl, sim_kw=None, counts=(100, 37)):
    """the deck's species with particles from the start: counts[0] below z = 0, counts[1] above (unequal slabs), the
    injectors behind them"""
    from warpx_b200.engine import Simulation
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], solver=abi.SOLVER_NONE, dt=wl["dt"],
                     **(sim_kw or {}))
    lo = [sim.prob_lo[d] + sim.dx[d] * sim.box_lo[d] for d in range(3)]
    hi = [sim.prob_lo[d] + sim.dx[d] * (sim.box_hi[d] + 1) for d in range(3)]
    for k, s in enumerate(wl["species"]):
        rng = np.random.default_rng(100 + k)
        n = sum(counts)
        P = dict(x=rng.uniform(-3.9, 3.9, n), y=rng.uniform(-3.9, 3.9, n),
                 z=np.concatenate([rng.uniform(-3.9, -0.1, counts[0]), rng.uniform(0.1, 3.9, counts[1])]),
                 w=np.ones(n), ux=np.zeros(n), uy=np.zeros(n), uz=np.zeros(n))
        own = np.ones(n, dtype=bool)
        for d, c in enumerate(("x", "y", "z")):
            own &= (P[c] >= lo[d]) & (P[c] < hi[d])
        sim.add_species(s["name"], s["q"], s["m"], *[np.ascontiguousarray(P[c][own]) for c in NAMES],
                        capacity=s["capacity"] + n)
    for s in wl["species"]:
        sim.add_flux_injection(s["name"], abi.make_flux_injector(**s["flux"]))
    return sim


@pytest.mark.parametrize("nb", [(1, 1, 2), (2, 2, 1)])
def test_bricks_on_species_with_particles(L, cuda, nb):
    """Species that hold particles from the start, unequally over the bricks: every rank's id counter starts at the
    global count, so the injected ids equal the single box's, and no id occurs twice."""
    import test_gpu_multirank as mr
    wl = _small_deck()
    nsp, n0 = len(wl["species"]), 137
    single = _seeded(wl)
    single.Evolve(2)
    want = [single.species_numpy(isp, sort_by_id=True) for isp in range(nsp)]
    want_next = [single.species_next_id(isp) for isp in range(nsp)]
    single.close()

    def rank(r, dist):
        sim = _seeded(wl, dict(dist=dist, nb=nb))
        counts = [sim.species[isp].np for isp in range(nsp)]
        sim.Evolve(2)
        return [sim.species_numpy(isp) for isp in range(nsp)], [sim.species_next_id(isp) for isp in range(nsp)], counts
    parts = mr.run_ranks(nb[0] * nb[1] * nb[2], rank)
    assert len({tuple(p[2]) for p in parts}) > 1                       # the ranks hold different numbers of particles
    for r in range(len(parts)):
        assert parts[r][1] == want_next
    got = _union([p[0] for p in parts])
    for g, w in zip(got, want):
        assert np.unique(g["id"]).size == g["id"].size
        gi, wi = (g["id"] >= n0) & (g["id"] < 1 << 40), w["id"] >= n0
        assert gi.sum() > 0 and np.array_equal(g["id"][gi], w["id"][wi])
        for k in ("w", "ux", "uy", "uz"):
            assert np.array_equal(g[k][gi].view(np.int64), w[k][wi].view(np.int64)), k


def test_restart_on_two_slabs_equals_the_straight_run(L, cuda, tmp_path):
    """N steps on 2 slabs along z, a checkpoint, a restart on 2 slabs, N more steps: the ids of the straight single-box
    run of 2N steps, each once; weights and momenta bit for bit, positions to 1e-13 of the domain."""
    import test_gpu_multirank as mr
    from warpx_b200 import diagnostics
    from warpx_b200.engine import Simulation
    wl = _small_deck()
    nsp, N, nb = len(wl["species"]), 2, (1, 1, 2)
    straight = build(wl)
    straight.Evolve(2 * N)
    want = [straight.species_numpy(isp, sort_by_id=True) for isp in range(nsp)]
    want_next = [straight.species_next_id(isp) for isp in range(nsp)]
    straight.close()
    prefix = str(tmp_path / "chk")

    def rank(r, dist):
        dist = _Gathering(dist)
        first = build(wl, dict(dist=dist, nb=nb))
        first.Evolve(N)
        root = diagnostics.write_checkpoint(first, prefix, N)
        first.close()
        sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], solver=abi.SOLVER_NONE,
                         dt=wl["dt"], dist=dist, nb=nb)
        diagnostics.read_checkpoint(sim, root, capacity={s["name"]: s["capacity"] for s in wl["species"]})
        for s in wl["species"]:
            sim.add_flux_injection(s["name"], abi.make_flux_injector(**s["flux"]))
        sim.Evolve(N)
        return [sim.species_numpy(isp) for isp in range(nsp)], [sim.species_next_id(isp) for isp in range(nsp)]
    parts = mr.run_ranks(2, rank)
    for p in parts:
        assert p[1] == want_next
    got = _union([p[0] for p in parts])
    for g, w in zip(got, want):
        assert np.unique(g["id"]).size == g["id"].size
        assert np.array_equal(g["id"], w["id"])
        for k in ("w", "ux", "uy", "uz"):
            assert np.array_equal(g[k].view(np.int64), w[k].view(np.int64)), k
        for k in ("x", "y", "z"):
            assert np.abs(g[k] - w[k]).max() <= 1e-13 * 8.0, k


def test_restart_equals_the_straight_run(cuda, tmp_path):
    from warpx_b200 import diagnostics
    from warpx_b200.engine import Simulation
    wl = _small_deck()
    N = 2
    straight = build(wl)
    straight.Evolve(2 * N)
    want = [straight.species_numpy(isp, sort_by_id=True) for isp in range(len(wl["species"]))]
    first = build(wl)
    first.Evolve(N)
    root = diagnostics.write_checkpoint(first, str(tmp_path / "chk"), N)
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], solver=abi.SOLVER_NONE, dt=wl["dt"])
    diagnostics.read_checkpoint(sim, root, capacity={s["name"]: s["capacity"] * 2 for s in wl["species"]})
    for s in wl["species"]:
        sim.add_flux_injection(s["name"], abi.make_flux_injector(**s["flux"]))
    sim.Evolve(N)
    got = [sim.species_numpy(isp, sort_by_id=True) for isp in range(len(wl["species"]))]
    _same(got, want)
    for g in got:
        assert np.unique(g["id"]).size == g["id"].size


def test_electromagnetic_run_and_launches(L, cuda):
    from warpx_b200.engine import Simulation

    def run(tmin):
        sim = Simulation((32, 32, 32), (0.0, 0.0, 0.0), (32e-6, 32e-6, 32e-6), nox=3)
        sim.add_empty_species("e", 300000, q=-1.602176634e-19, m=9.1093837015e-31)
        if tmin is not None:
            sim.add_flux_injection("e", abi.make_flux_injector(8.0, 4e-6, "z", 1, flux=1e30, u_m=(0.0, 0.0, 0.05),
                                                               u_th=(0.01, 0.01, 0.01), flux_tmin=tmin, seed=5))
        sim.Evolve(1)
        n0 = L.pic_launch_count()
        sim.Evolve(6)
        return sim, L.pic_launch_count() - n0
    sim, _ = run(0.0)
    assert sim.species[0].np > 6 * 32 * 32 * 8 * 0.9
    for c in range(9):
        assert np.all(np.isfinite(sim.field_numpy(c)[1]))
    assert sim.field_energy()[0] > 0
    _, without = run(None)
    _, closed = run(1.0)                      # the window opens after the run: the stage launches nothing
    print("LAUNCHES", json.dumps(dict(without_injector=without, injector_outside_window=closed)))
    assert closed == without
