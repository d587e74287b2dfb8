"""CPU test of bench.py's control flow (argument handling, stage timing plumbing, e2e leg, explicit teardown, CPU leg,
the JSON line and its keys) with the CUDA pieces replaced by stand-ins: torch.cuda.* are stubs, Simulation is the host
harness's (the product library compiled for the host under the SIMT emulator).  It checks that the benchmark script
runs end to end and prints ONE well-formed line -- nothing about speed."""
import json
import sys
import types

import pytest


class _Event:
    def __init__(self, enable_timing=True):
        pass

    def record(self):
        pass

    def elapsed_time(self, other):
        return 2.0


def test_bench_engine_arm_prints_one_complete_line(monkeypatch, capfd, tmp_path):
    import torch
    from host_harness import harness
    import bench
    import warpx_b200.engine as eng
    import warpx_b200.lib as piclib
    Host = harness.host_simulation_class()
    monkeypatch.setattr(eng, "Simulation", Host)
    monkeypatch.setattr(piclib, "lib", harness.host_library)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "set_device", lambda *_: None)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *_: None)
    monkeypatch.setattr(torch.cuda, "empty_cache", lambda: None)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    real_tensor = torch.tensor
    monkeypatch.setattr(torch, "tensor", lambda *a, **k: real_tensor(*a, **{kk: v for kk, v in k.items() if kk != "device"}))
    monkeypatch.setattr(bench, "start_watchdog", lambda rank: None)
    # the host library has no CUDA events: feed the stage table the roofline code expects
    monkeypatch.setattr(Host, "enable_stage_timing", lambda self, on=True: None)
    monkeypatch.setattr(Host, "stage_ms", lambda self: {"gather_push": (1.0, 2), "deposit": (2.0, 2), "evolve_b": (0.1, 4),
                                                      "evolve_e": (0.1, 2), "sort": (0.5, 1)})
    evolved = []
    real_evolve = Host.Evolve
    monkeypatch.setattr(Host, "Evolve", lambda self, n, **k: (evolved.append(n), real_evolve(self, n, **k))[1])
    dump = tmp_path / "dump"
    monkeypatch.setattr(sys, "argv", ["bench.py", "--cells", "16", "--steps", "2", "--warmup", "3", "--spinup", "1",
                                      "--cpu-cells", "16", "--cpu-steps", "1", "--deposit-mode", "7",
                                      "--dump-outputs", str(dump)])
    monkeypatch.setattr(bench.os, "_exit", lambda code: (_ for _ in ()).throw(SystemExit(code)))
    monkeypatch.setattr(bench.atexit, "_run_exitfuncs", lambda: None)      # not pytest's own exit handlers
    with pytest.raises(SystemExit) as e:
        bench.main()
    assert e.value.code == 0
    out = [ln for ln in capfd.readouterr().out.splitlines() if ln.startswith("{")]
    assert len(out) == 1
    line = json.loads(out[0])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline"):
        assert key in line, key
    assert line["n_gpus"] == 1 and line["steps"] == 2 and line["dtype"] == "f64" and line["vs_baseline"] is None
    assert line["roofline"]["kernel"] in ("deposit", "gather_push") and 0 < line["roofline"]["frac"]
    assert line["e2e"]["h2d_bytes_per_step"] > 0 and line["e2e"]["d2h_bytes_per_step"] == 16
    assert line["cpu_baseline"]["value"] and line["cpu_baseline"]["cores"] >= 1
    assert "workload" in line["config"] and line["config"]["deposit_mode"] == 7
    assert evolved[:3] == [1, 3, 2]                  # spin-up, warm-up, then exactly --steps timed steps
    # --dump-outputs: what the timed steps computed, float64, a fixed sample, well under 64 MB
    import numpy as np
    from warpx_b200 import abi
    names = ["field_energy", "particle_id"] + list(abi.COMP_NAMES) + ["particle_" + k for k in ("x", "y", "z", "w", "ux", "uy", "uz")]
    assert sorted(p.name for p in dump.iterdir()) == sorted(n + ".npy" for n in names)
    arrs = {n: np.load(dump / (n + ".npy")) for n in names}
    assert all(a.dtype == np.float64 for a in arrs.values())
    assert sum(a.nbytes for a in arrs.values()) <= 64 << 20
    assert np.allclose(arrs["field_energy"], line["field_energy_J"], rtol=1e-12)
    assert arrs["Ex"].size == 16 * 17 * 17 and np.all(np.diff(arrs["particle_id"]) > 0)     # valid points, nodal in y, z
    assert arrs["particle_x"].size == arrs["particle_id"].size == 16 ** 3 * 8
    harness.host_library().pic_set_deposit_mode(0)


def test_bench_reference_arm_prints_one_line(monkeypatch, capfd):
    import bench
    monkeypatch.setattr(sys, "argv", ["bench.py", "--impl", "reference", "--cpu-cells", "16", "--steps", "2", "--warmup", "1"])
    monkeypatch.setattr(bench.os, "_exit", lambda code: (_ for _ in ()).throw(SystemExit(code)))
    monkeypatch.setattr(bench.atexit, "_run_exitfuncs", lambda: None)      # not pytest's own exit handlers
    with pytest.raises(SystemExit):
        bench.main()
    out = [ln for ln in capfd.readouterr().out.splitlines() if ln.startswith("{")]
    assert len(out) == 1
    line = json.loads(out[0])
    assert line["impl"] == "reference" and line["value"] > 0 and line["e2e"]["value"] == line["value"]
    assert line["cpu_baseline"]["kind"] in ("port", "reference-leaves+port")
