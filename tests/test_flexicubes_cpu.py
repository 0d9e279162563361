"""FlexiCubes without a GPU: the case table (scripts/gen_fc_table.py -> csrc/fc_table.cuh) against the reference's
tables, the torch oracle (oracle/fc_oracle.py) in fp32 and fp64 against the reference's own outputs and gradients
(tests/golden/ref_flexicubes.npz), and the closed-form voxel grid against the reference's grid."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle import fc_oracle as O

sys.path.insert(0, os.path.join(ROOT, "scripts"))
import gen_fc_table as G  # noqa: E402

Z = np.load(os.path.join(GOLDEN, "ref_flexicubes.npz"))
CASES = ["sphere", "random", "boundary", "zeros", "inside", "outside"]


def test_generator_reproduces_the_committed_header():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "gen_fc_table.py"), "--check"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


def test_derived_tables_equal_the_references():
    groups, check = G.build_table()
    assert np.array_equal(np.array([len(g) for g in groups]), Z["num_vd_table"])
    assert np.array_equal(np.array(check), Z["check_table"])
    dmc = Z["dmc_table"]
    for c in range(256):
        ref = sorted(tuple(sorted(int(e) for e in row if e != -1)) for row in dmc[c][:Z["num_vd_table"][c]])
        assert sorted(tuple(g) for g in groups[c]) == ref, c


def test_ambiguity_rows_follow_the_rule():
    groups, check = G.build_table()
    flagged = [c for c in range(256) if check[c][0]]
    assert len(flagged) == 36
    assert {bin(c).count("1") for c in flagged} == {5, 6}
    for c in flagged:
        assert len(groups[c]) == 1 and check[c][4] == 255 - c
        assert len(groups[255 - c]) == 2          # the complement separates the two inside corners


def test_fixture_random_case_hits_both_inversions():
    n5, n6 = Z["random/inversions"]
    assert n5 > 0 and n6 > 0


@pytest.mark.parametrize("tag,res", [("6", 6), ("4_7_5", (4, 7, 5))])
def test_closed_form_grid_equals_the_references(tag, res):
    from gs_b200.isosurface import FlexiCubes
    v, c = FlexiCubes(device="cpu").construct_voxel_grid(res)
    assert v.dtype == torch.float32 and c.dtype == torch.int64
    assert np.array_equal(v.numpy().view(np.uint32), Z[f"grid/{tag}/verts"].view(np.uint32))
    assert np.array_equal(c.numpy(), Z[f"grid/{tag}/cubes"])


@pytest.mark.parametrize("res", [100, 127, 128, 256])
def test_closed_form_grid_digests(res):
    from gs_b200.isosurface import voxel_grid
    v, c = voxel_grid(res, "cpu")
    assert [v.shape[0], c.shape[0]] == Z[f"grid/{res}/shapes"].tolist()
    assert hashlib.sha256(v.numpy().tobytes()).hexdigest() == Z[f"grid/{res}/sha256"][0]
    assert hashlib.sha256(c.numpy().tobytes()).hexdigest() == Z[f"grid/{res}/sha256"][1]


def test_construct_voxel_grid_returns_fresh_tensors():
    from gs_b200.isosurface import FlexiCubes
    fc = FlexiCubes(device="cpu")
    a, _ = fc.construct_voxel_grid(4)
    a *= 2
    b, _ = fc.construct_voxel_grid(4)
    assert float(b.abs().max()) == 0.5


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_reference(name, dtype):
    res, x, s, w = O.fixture_inputs(Z, name)
    for ws, given, training in O.VARIANTS:
        fn = lambda x_, s_, b, a, g: O.flexicubes(x_, s_, res, b, a, g, training=bool(training), weight_scale=ws,
                                                   dtype=dtype)
        v, f, L, (keys,), grads = O.run_with_grads(fn, x, s, w, given, Z)
        O.assert_matches_fixture(Z, f"{name}/{ws}/{given}/{training}", v, f, L, keys, grads)
