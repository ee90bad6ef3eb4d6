"""rtg_map_transform on the GPU: per-anchor rigid transforms of the map against the float64 oracle, rows that must stay
bit-identical, render invariance through the rasterizer (the end-to-end check of the SH rotation's signs and of the
quaternion), composition of two corrections, and the full map size."""
import numpy as np
import pytest
import torch

import helpers
from oracle import maptransform_oracle as mo
from oracle.splat_oracle import OracleRender
from rtg_slam_b200 import mapsurgery, scene

pytestmark = pytest.mark.gpu


def _map(P, K, seed, frac_unanchored=0.05, frac_out=0.02, frac_unmoved=0.1):
    """Seeded map and K anchor corrections (<= 45 deg, <= 2 m); some anchors -1, some out of range, some unmoved."""
    rng = np.random.default_rng(seed)
    f = np.float32
    params = {"xyz": rng.uniform(-4, 4, (P, 3)).astype(f),
              "rotation": (rng.normal(size=(P, 4)) * rng.uniform(0.3, 3.0, (P, 1))).astype(f),
              "normal": mo.unit_dirs(P, rng).astype(f),
              "features_rest": rng.normal(0, 0.5, (P, 15, 3)).astype(f),
              "features_dc": rng.normal(size=(P, 1, 3)).astype(f)}
    old = np.stack([mo.random_pose(rng) for _ in range(K)])
    new = np.stack([mo.corrected_pose(rng, o) for o in old])
    unmoved = rng.uniform(size=K) < frac_unmoved
    new[unmoved] = old[unmoved]
    anchor = rng.integers(0, K, P).astype(np.int32)
    u = rng.uniform(size=P)
    anchor[u < frac_unanchored] = -1
    out = (u >= frac_unanchored) & (u < frac_unanchored + frac_out)
    anchor[out] = np.where(rng.uniform(size=int(out.sum())) < 0.5, rng.integers(K, 2 * K + 5, int(out.sum())),
                           rng.integers(-1000, -1, int(out.sum()))).astype(np.int32)
    return params, anchor, old, new


def _to_dev(params, dev, sh_rest=15):
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in params.items()}
    if sh_rest < 15:
        t["features_rest"] = t["features_rest"][:, :sh_rest].contiguous()
    if sh_rest == 0:
        del t["features_rest"]
    return t


def _check_against_oracle(got, src, exp, moved, anchor, old, new, rows, scale=1.0):
    """Bounds of the issue: xyz 2e-6 (1 + |x| + |t|), quaternion 2e-6 |q|, normal 2e-6, SH 1e-5 ||f_l|| per band and
    channel; `scale` widens them for chained calls."""
    a = anchor[rows]
    t = np.zeros(len(rows))
    for k in np.unique(a[moved]):
        t[moved & (a == k)] = np.linalg.norm(mo.anchor_transform(old[k], new[k])[2])
    x0 = src["xyz"][rows].astype(np.float64)
    err = np.abs(got["xyz"] - exp["xyz"]).max(1)
    assert (err <= scale * 2e-6 * (1 + np.linalg.norm(x0, axis=1) + t)).all(), err.max()
    q0 = np.linalg.norm(src["rotation"][rows].astype(np.float64), axis=1)
    assert (np.abs(got["rotation"] - exp["rotation"]).max(1) <= scale * 2e-6 * q0).all()
    assert np.abs(got["normal"] - exp["normal"]).max() <= scale * 2e-6
    if "features_rest" in got:
        f0 = src["features_rest"][rows].astype(np.float64)
        M = got["features_rest"].shape[1] + 1
        for l, b in mo.BANDS.items():
            if b.stop > M:
                continue
            rb = slice(b.start - 1, b.stop - 1)
            bound = scale * 1e-5 * np.linalg.norm(f0[:, rb], axis=1)          # (n, 3): per row and channel
            assert (np.abs(got["features_rest"][:, rb] - exp["features_rest"][:, rb]).max(1) <= bound).all(), l


@pytest.fixture(scope="module")
def case200k():
    params, anchor, old, new = _map(200_000, 1000, seed=1)
    exp, moved, n_skipped = mo.transform({k: v for k, v in params.items() if k != "features_dc"}, anchor, old, new)
    return params, anchor, old, new, exp, moved, n_skipped


@pytest.mark.parametrize("sh_rest", [0, 3, 8, 15])
def test_kernel_matches_the_oracle_and_leaves_other_rows_bit_identical(cuda_device, case200k, sh_rest):
    params, anchor, old, new, exp, moved, n_skipped = case200k
    t = _to_dev(params, cuda_device, sh_rest)
    before = {k: v.clone() for k, v in t.items()}
    an = torch.from_numpy(anchor).to(cuda_device)
    if sh_rest == 8:
        an = an[:, None]                                                     # the (P, 1) layout of _add_tick
    n = mapsurgery.transform(t, an, old, new)
    assert n.is_cuda and n.dtype == torch.int64
    assert int(n.item()) == n_skipped > 0
    got = {k: v.cpu().numpy().astype(np.float64) for k, v in t.items()}
    rows = np.arange(len(anchor))
    e = dict(exp)
    if sh_rest:
        e["features_rest"] = exp["features_rest"][:, :sh_rest]
    _check_against_oracle(got, params, e, moved, anchor, old, new, rows)
    keep = torch.from_numpy(~moved).to(cuda_device)
    for k in t:
        assert torch.equal(t[k][keep], before[k][keep]), k                    # unmoved, unanchored, out of range
    assert torch.equal(t["features_dc"], before["features_dc"])
    assert moved.sum() > 0.8 * len(anchor)


def _offset_rows(t):
    """A contiguous copy of `t` that starts one float into a larger buffer (4-byte, not 16-byte aligned), and the buffer."""
    buf = torch.full((t.numel() + 5,), 7.0, dtype=t.dtype, device=t.device)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    return v, buf


@pytest.mark.parametrize("layout", ["offset", "no_normal"])
def test_unaligned_rows_and_missing_normal(cuda_device, case200k, layout):
    """The word-by-word path of arrays that are not 16-byte aligned, and a map without cached normals."""
    params, anchor, old, new, exp, moved, n_skipped = case200k
    t = _to_dev(params, cuda_device)
    bufs = {}
    if layout == "offset":
        for k in ("xyz", "rotation", "normal", "features_rest"):
            t[k], bufs[k] = _offset_rows(t[k])
            assert t[k].data_ptr() % 16 == 4 and t[k].is_contiguous()
    else:
        normal_before = t.pop("normal").clone()
    before = {k: v.clone() for k, v in t.items()}
    n = mapsurgery.transform(t, torch.from_numpy(anchor).to(cuda_device), old, new)
    assert int(n.item()) == n_skipped
    got = {k: v.cpu().numpy().astype(np.float64) for k, v in t.items()}
    if layout == "no_normal":
        got["normal"] = exp["normal"]
        assert "normal" not in t and normal_before.shape[0] == len(anchor)
    _check_against_oracle(got, params, exp, moved, anchor, old, new, np.arange(len(anchor)))
    keep = torch.from_numpy(~moved).to(cuda_device)
    for k in t:
        assert torch.equal(t[k][keep], before[k][keep]), k
    for k, buf in bufs.items():                                                    # nothing written outside the rows
        assert float(buf[0]) == 7.0 and bool((buf[1 + t[k].numel():] == 7.0).all()), k


def test_no_anchor_poses_counts_every_anchored_row(cuda_device):
    """K == 0: nothing moves; every anchor other than -1 is out of range and counted."""
    params, anchor, _, _ = _map(10_000, 50, seed=3)
    t = _to_dev(params, cuda_device)
    before = {k: v.clone() for k, v in t.items()}
    empty = np.zeros((0, 4, 4))
    n = mapsurgery.transform(t, torch.from_numpy(anchor).to(cuda_device), empty, empty)
    assert int(n.item()) == int((anchor != -1).sum()) > 0
    for k in t:
        assert torch.equal(t[k], before[k]), k


def test_non_tensor_attributes_raise_type_error(cuda_device):
    old = np.eye(4)[None]
    new = old.copy()
    new[0, 0, 3] = 1.0
    for key in ("rotation", "normal", "features_rest"):
        p = {"xyz": torch.zeros(4, 3, device=cuda_device), "rotation": torch.zeros(4, 4, device=cuda_device),
             key: [[0.0] * 4] * 4}
        with pytest.raises(TypeError):
            mapsurgery.transform(p, torch.zeros(4, dtype=torch.int32, device=cuda_device), old, new)


def test_render_is_invariant_under_a_rigid_move_of_map_and_camera(cuda_device):
    """One anchor's 30 deg / 1 m correction T applied to every Gaussian and c2w' = T c2w to the camera: colour, depth and
    T_map agree under compare_outputs, the index maps agree outside threshold ties, the normal map is R times the old one;
    without rotating features_rest the colour misses the tolerance by at least 10x.

    The base camera is turned away from the room's axes: seen from the identity pose the back wall is fronto-parallel, so
    its coplanar surfels share one depth key, the sort keeps them in index order, and after any rotation float32 rounding
    breaks those ties differently (z-fighting between overlapping surfels), which is not what this test is about."""
    base = scene.small_pose((7.0, -5.0, 3.0), (0.1, -0.05, 0.2))
    cam = scene.make_camera("replica", c2w=base)
    g = scene.surfel_room(100_000, seed=3)
    rng = np.random.default_rng(5)
    # the view-dependent part of the colour as large as the DC part: RMS 0.33 over directions against 0.29
    g["shs"][:, 1:] = rng.normal(0, 0.3, g["shs"][:, 1:].shape).astype(np.float32)
    axis = np.array([0.3, -0.8, 0.52]) / np.linalg.norm([0.3, -0.8, 0.52])
    T = np.eye(4)
    T[:3, :3] = mo.Rotation.from_rotvec(axis * np.deg2rad(30.0)).as_matrix()
    T[:3, 3] = np.array([0.6, -0.48, 0.64])                                          # 1 m
    cam2 = scene.make_camera("replica", c2w=T @ base)

    def moved(with_rest):
        p = {"xyz": torch.from_numpy(g["xyz"]).to(cuda_device), "rotation": torch.from_numpy(g["rotations"]).to(cuda_device),
             "normal": torch.from_numpy(g["normal"]).to(cuda_device)}
        if with_rest:
            p["features_rest"] = torch.from_numpy(np.ascontiguousarray(g["shs"][:, 1:])).to(cuda_device)
        anchor = torch.zeros(len(g["xyz"]), dtype=torch.int32, device=cuda_device)
        assert int(mapsurgery.transform(p, anchor, np.eye(4)[None], T[None]).item()) == 0
        h = dict(g)
        h["xyz"], h["rotations"], h["normal"] = (p[k].cpu().numpy() for k in ("xyz", "rotation", "normal"))
        if with_rest:
            h["shs"] = np.concatenate([g["shs"][:, :1], p["features_rest"].cpu().numpy()], 1)
        return h

    ref = helpers.run_ours(cam, g, cuda_device)
    h = moved(True)
    out = helpers.run_ours(cam2, h, cuda_device)
    # threshold ties of either render (the float32 oracle's tie class, as every rasterizer comparison here uses it)
    tie = OracleRender(cam, g, precision="f32", tie_eps=1e-4).tie | OracleRender(cam2, h, precision="f32", tie_eps=1e-4).tie
    st = helpers.compare_outputs(out, ref, tie=tie, label="moved map and camera")
    H, W = cam.height, cam.width
    same = (out["hit_color"][0] == ref["hit_color"][0]) & (out["hit_depth"][0] == ref["hit_depth"][0])
    assert (~same & ~tie.astype(bool)).sum() <= 2e-4 * H * W, st
    hit = same & (ref["hit_depth"][0] >= 0)
    assert hit.sum() > 0.5 * H * W
    nm_old = g["normal"][ref["hit_depth"][0][hit]].astype(np.float64)
    nm_new = h["normal"][out["hit_depth"][0][hit]].astype(np.float64)
    np.testing.assert_allclose(nm_new, nm_old @ T[:3, :3].T, rtol=0, atol=2e-6)
    # negative control: the same move without rotating the SH coefficients
    bad = helpers.run_ours(cam2, moved(False), cuda_device)
    same_b = (bad["hit_color"][0] == ref["hit_color"][0]) & (bad["hit_depth"][0] == ref["hit_depth"][0])
    miss = np.abs(bad["color"].astype(np.float64) - ref["color"]).max(0)[same_b].max()
    assert miss >= 10 * 1e-4, miss


def test_two_corrections_compose(cuda_device):
    params, anchor, old, new = _map(200_000, 1000, seed=2)
    rng = np.random.default_rng(9)
    mid = np.stack([mo.corrected_pose(rng, o) for o in old])
    mid[np.all(old == new, axis=(1, 2))] = old[np.all(old == new, axis=(1, 2))]
    a = torch.from_numpy(anchor).to(cuda_device)
    two = _to_dev(params, cuda_device)
    mapsurgery.transform(two, a, old, mid)
    mapsurgery.transform(two, a, mid, new)
    one = _to_dev(params, cuda_device)
    mapsurgery.transform(one, a, old, new)
    moved = np.asarray([not np.array_equal(old[k], new[k]) if 0 <= k < len(old) else False for k in anchor])
    rows = np.nonzero(moved)[0]
    got = {k: v.cpu().numpy().astype(np.float64)[rows] for k, v in two.items()}
    exp = {k: v.cpu().numpy().astype(np.float64)[rows] for k, v in one.items()}
    _check_against_oracle(got, params, exp, np.ones(len(rows), bool), anchor, old, new, rows, scale=2.0)


def test_full_map_size_against_the_oracle_on_a_sample(cuda_device):
    params, anchor, old, new = _map(1_000_000, 3000, seed=4)
    t = _to_dev(params, cuda_device)
    n = mapsurgery.transform(t, torch.from_numpy(anchor).to(cuda_device), old, new)
    rows = np.sort(np.random.default_rng(11).choice(len(anchor), 20_000, replace=False))
    src = {k: v for k, v in params.items() if k != "features_dc"}
    exp, moved, n_skipped = mo.transform(src, anchor, old, new, rows=rows)
    assert int(n.item()) == n_skipped
    idx = torch.from_numpy(rows).to(cuda_device)
    got = {k: t[k][idx].cpu().numpy().astype(np.float64) for k in src}
    _check_against_oracle(got, params, exp, moved, anchor, old, new, rows)
    for k in src:
        np.testing.assert_array_equal(got[k][~moved], params[k][rows][~moved])
