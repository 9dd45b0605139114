"""CPU tier: the __host__ __device__ bodies of the CUDA localization kernels, executed by the host emulation
harness (tests/emu), against the oracle -- bit-exact voxel keys, octree shape, match sets, normal equations, state."""
import numpy as np

from immesh_b200 import api
from lio_common import run_degenerate_map_parity, run_stream_parity


def test_avia_stream_bit_exact(emu_lib):
    stats = run_stream_parity(emu_lib, "avia", api.AVIA, n_scans=12, seed=0)
    assert stats[-1]["n_match"] > stats[0]["n_match"]          # the map densifies
    assert all(s["pos_err"] < 0.05 for s in stats)             # and the filter tracks the trajectory


def test_hdl64_octree_depth_bit_exact(emu_lib):
    # velodyne.yaml: 3 m root voxels, 4 layers, 1000-point nodes -> exercises cut_octo_tree recursion and freezing
    stats = run_stream_parity(emu_lib, "hdl64", api.VELODYNE, n_scans=4, seed=1, n_points=32768)
    assert stats[-1]["n_match"] > 500


def test_other_residual_bodies_bit_exact(emu_lib):
    # The default emulation runs the 8-lanes-per-point match + the terms step (k_match, k_terms).  Mode 2 is k_match's choice for large
    # scans (one lane per point through the same code), mode 0 the single-step body (k_residual, used by immesh_lio_residual_build).
    # All must reproduce the oracle's walk.
    try:
        for mode in (2, 0):
            emu_lib.emu_lio_set_split(mode)
            run_stream_parity(emu_lib, "avia", api.AVIA, n_scans=5, seed=3)
            run_stream_parity(emu_lib, "hdl64", api.VELODYNE, n_scans=3, seed=2, n_points=16384)
    finally:
        emu_lib.emu_lio_set_split(1)


def test_degenerate_root_voxels_bit_exact(emu_lib):
    # pole, repeated point, exact plane, root and child borders at negative coordinates: NaN-aware, each case asserted
    run_degenerate_map_parity(emu_lib)
