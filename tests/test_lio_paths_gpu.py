"""GPU tier: localization paths the synthetic streams of the other tests do not reach, stage by stage against the oracle.

    k_match, 8 lanes per point     n <= 256 * SMs (the grid is 8 blocks of 128 per SM; 8 lanes while n * 8 <= 2 * threads)
    k_match, 1 lane per point      n >  256 * SMs
The threshold is read from the device, so the boundary pair (exactly 256 * SMs and one point more) is right on any GPU.  Also:
degenerate root voxels through buildVoxelMap and one state estimation, and a 1 M-point scan through the pipelined path at
bench.py's C5 settings."""
import pytest

from immesh_b200 import api, synth
from lio_common import run_degenerate_map_parity, run_stream_parity
from parity_gate import pipeline_parity

pytestmark = pytest.mark.gpu


def _one_lane_threshold():
    import torch
    return 256 * torch.cuda.get_device_properties(0).multi_processor_count


def test_k_match_both_lane_modes_and_the_boundary(cuda_lib):
    """Scan 1 above the threshold (1 lane per point), scan 2 truncated to exactly the threshold (8 lanes), scan 3 to one point
    more (1 lane): matches, normal equations per iteration, state and map bit-exact after every scan."""
    thr = _one_lane_threshold()
    cfg = api.LioConfig(filter_size_surf=0.1)
    sensor, scans = synth.make_stream("avia100k", 2, seed=0, leaf=0.1, ext_T=cfg.ext_T)
    assert scans[1]["body_ds"].shape[0] > thr + 1, "the stream must reach the 1-lane path"
    stats = run_stream_parity(cuda_lib, "avia100k", cfg, n_scans=4, seed=0, body_len={2: thr, 3: thr + 1})
    assert stats[0]["n"] > thr + 1 and stats[1]["n"] == thr and stats[2]["n"] == thr + 1
    assert min(s["n_match"] for s in stats) > 1000


def test_degenerate_root_voxels_map_and_estimation(cuda_lib):
    """pole, repeated point, exact plane, root and child borders at negative coordinates (lio_common.degenerate_root_voxels
    states what the reference computes for each): buildVoxelMap and one state estimation, NaN-aware, each case asserted"""
    run_degenerate_map_parity(cuda_lib)


def test_c5_shape_scan_pipelined(cuda_lib):
    """one 1 M-point scan through the pipelined path with bench.py's own C5 settings (taken from bench.workloads(), so the two
    cannot drift): a 1 M-point transform and upload, about 10 k append candidates (every ~100th point), 0.2 m voxels"""
    import bench
    w = bench.workloads()["C5"]
    sensor, scans = synth.make_stream(w["kind"], 2, seed=11, leaf=w["lio"].filter_size_surf, ext_T=w["lio"].ext_T)
    assert scans[1]["body_full"].shape[0] > 1000000
    rep = pipeline_parity(cuda_lib, w["lio"], w["mesh"], scans, 1, oracle_threads=(8, 8))
    assert rep["ok"], rep
    assert rep["vertices"][0] > 5000
