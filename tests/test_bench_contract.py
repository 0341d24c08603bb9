"""bench.py --impl reference runs on CPU: check the JSON contract of the reference arm (and, by
construction, of the keys the GPU arm shares) without a GPU."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_json_line():
    env = dict(os.environ, B200TSDF_REF_THREADS="2")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["unit"] == "frames/s" and line["higher_is_better"] is True
    assert line["metric"].startswith("integrateCloud frames/s") and line["n_gpus"] == 1 and line["steps"] == 1 and line["warmup"] == 1
    assert line["value"] > 0 and line["e2e"]["value"] == line["value"] and line["e2e"]["h2d_bytes_per_step"] == 0
    cb = line["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] == 2 and cb["value"] == line["value"]
    assert "workload" in line["config"] and line["data"] == "synthetic" and line["vs_baseline"] is None


def test_other_ranks_of_the_reference_arm_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=120, env=env, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.strip() == ""


@pytest.mark.parametrize("name", ["h100_bench.json"])
def test_committed_gpu_bench_line_has_every_contract_key(name):
    """profiles/h100_bench.json is the line `python bench.py --gpus 1 --steps 20 --warmup 3` printed on one H100 SXM (80 GB HBM3,
    400 W power limit): check its shape against the contract."""
    d = json.load(open(os.path.join(ROOT, "profiles", name)))
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline"):
        assert k in d, k
    assert d["unit"] == "frames/s" and d["n_gpus"] == 1 and d["warmup"] >= 3 and d["higher_is_better"] is True and d["vs_baseline"] is None
    assert "workload" in d["config"] and "l2" in d["config"] and d["data"] == "synthetic" and d["dtype"] == "f32"
    assert set(d["clocks"]) >= {"sm_mhz", "sm_max_mhz", "reasons"} and not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    e = d["e2e"]
    # bytes that crossed PCIe per 32-frame step: the caller's 32-byte points (round 1), or the 16-byte pixels the host packed them to
    packed = bool(e.get("host_pack", {}).get("enabled"))
    assert e["unit"] == "frames/s" and 0 < e["value"] < d["value"] and e["h2d_bytes_per_step"] == 32 * 640 * 480 * (16 if packed else 32) and e["d2h_bytes_per_step"] > 0
    if packed:
        assert e["host_pack"]["input_bytes_per_step"] == 32 * 640 * 480 * 32 and e["host_pack"]["threads"] >= 1
    r = d["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert r["traffic"] > 0 if r["traffic_source"] != "not measured" else r["traffic"] is None
    c = d["cpu_baseline"]
    assert c["kind"] in ("reference", "port") and c["cores"] >= 1 and c["value"] > 0 and c["unit"] == "frames/s" and c["sample"]
    assert d["gpu_launches"] == 4 * 32 * d["steps"]                      # four kernels per frame, 32 frames per step
    assert abs(d["value"] - 32 / (d["ms_per_step"] * 1e-3)) / d["value"] < 1e-6
    # one graph launch per 32-frame step, a batched roofline figure next to the event-timed one, the loaded-host leg
    assert d["graph_launches"] == d["steps"]
    b = r["batched"]
    assert b["frames_per_graph_launch"] == 32 and abs(b["frac"] - b["achieved"] / r["peak"]) < 1e-9 and b["frac"] >= r["frac"]
    hl = d["host_load_leg"]
    assert hl["unit"] == "frames/s" and len(hl["repeats"]) == 3 and abs(hl["value"] - sorted(hl["repeats"])[1]) < 1e-9
    assert hl["value"] > 0.9 * d["value"]                            # the device-resident rate does not depend on an idle host


def test_dump_outputs_writes_a_bounded_key_sampled_volume(tmp_path, monkeypatch):
    """bench.py --dump-outputs: float32/float64 .npy files, nodes chosen by their key alone (so two builds dump the same keys
    wherever they agree), and the node cap keeps the whole dump under 64 MB."""
    import importlib.util
    import types

    import numpy as np
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)

    class StubVolume:
        def __init__(self, keys, seed):
            rng = np.random.default_rng(seed)
            n = len(keys)
            self.d = {"keys": keys, "dw": rng.random((n, 2), dtype=np.float32), "split": rng.integers(0, 2, n).astype(np.uint8),
                      "rgb": rng.integers(0, 256, (n, 3)).astype(np.uint8)}

        def download_nodes(self):
            return self.d

        def stats(self):
            return types.SimpleNamespace(n_updates=11, n_node_visits=12, n_bricks=13, n_block_visits=14)

    rng = np.random.default_rng(0)
    n = 200_000
    keys = np.stack([rng.integers(5, 12, n), rng.integers(0, 2048, n), rng.integers(0, 2048, n), rng.integers(0, 2048, n)], 1).astype(np.int32)
    a, b = tmp_path / "a", tmp_path / "b"
    bench.dump_outputs(StubVolume(keys, 1), str(a))
    bench.dump_outputs(StubVolume(keys, 2), str(b))                 # same keys, different values
    names = {"node_keys", "node_sdf_weight", "node_split", "node_rgb", "volume_counts"}
    assert {p.stem for p in a.iterdir()} == names and all(p.suffix == ".npy" for p in a.iterdir())
    out = {k: np.load(a / f"{k}.npy") for k in names}
    assert all(v.dtype in (np.float32, np.float64) for v in out.values())
    m = len(out["node_keys"])
    assert 0.5 * n / bench.DUMP_SAMPLE < m < 2 * n / bench.DUMP_SAMPLE
    assert out["node_sdf_weight"].shape == (m, 2) and out["node_split"].shape == (m,) and out["node_rgb"].shape == (m, 3)
    assert np.array_equal(out["node_keys"], np.load(b / "node_keys.npy"))
    assert not np.array_equal(out["node_sdf_weight"], np.load(b / "node_sdf_weight.npy"))
    assert out["volume_counts"].tolist() == [n, 11, 12, 13, 14]
    # the cap: the first DUMP_MAX_NODES selected nodes in the engine's order, and at the real cap the dump stays under 64 MB
    per_node = sum(v.nbytes for k, v in out.items() if k != "volume_counts") / m
    assert bench.DUMP_MAX_NODES * per_node + out["volume_counts"].nbytes < 64 * 2**20
    monkeypatch.setattr(bench, "DUMP_MAX_NODES", 100)
    bench.dump_outputs(StubVolume(keys, 1), str(tmp_path / "c"))
    assert np.array_equal(np.load(tmp_path / "c" / "node_keys.npy"), out["node_keys"][:100])
