"""CPU tests of the mapping step under a keyframe exposure: float64 statements of the mapping loss and of the SSIM term
under an exposure (a, b), each pinned by central differences in a and b, and the host validation of
rtg_loss_mapping_exposure and rtg_ssim_loss_exposure (no CUDA work is reached)."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_pose_exposure_cpu import loss_statement, mapping_frame

EXPOSURES = [(0.0, 0.0), (0.2, 0.05), (-0.25, -0.03)]


def mapping_statement_inputs(use_mask):
    H, W = 23, 31
    gen = torch.Generator().manual_seed(5)
    render, depth, normal, depth_index, gt_color, gt_depth, gt_normal = mapping_frame(H, W, gen)
    n = H * W
    mask = (torch.rand(n, generator=gen) < 0.6) if use_mask else torch.ones(n, dtype=torch.bool)
    return (render.reshape(3, n), depth.reshape(n), depth_index.reshape(n), gt_color.permute(2, 0, 1).reshape(3, n),
            gt_depth.reshape(n), mask, normal.reshape(3, n), gt_normal.permute(2, 0, 1).reshape(3, n))


def mapping_statement(inputs, ab, normal_weight=0.1):
    """test_pose_exposure_cpu.loss_statement with the normal term and the exposure: rtg_loss_mapping_exposure's statement."""
    render, depth, hit, gt_color, gt_depth, mask, normal, gt_normal = inputs
    return loss_statement(render, depth, hit, gt_color, gt_depth, mask, 0.8, 1.0, 0.1, ab, normal=normal, gt_normal=gt_normal,
                          normal_weight=normal_weight)


def central(f, ab, h):
    """Central differences of the scalar f(a, b) in a and in b."""
    a, b = ab
    return np.array([(f((a + h, b)) - f((a - h, b))) / (2 * h), (f((a, b + h)) - f((a, b - h))) / (2 * h)])


@pytest.mark.parametrize("use_mask", [False, True])
@pytest.mark.parametrize("ab", EXPOSURES)
def test_mapping_loss_statement_under_an_exposure_matches_central_differences(ab, use_mask):
    inputs = mapping_statement_inputs(use_mask)
    parts, gC, gD, gN, gE = mapping_statement(inputs, ab)
    # L1 is piecewise linear in (a, b): a step well below the smallest |residual| stays on one piece
    render, gt_color, mask = inputs[0], inputs[3], inputs[5]
    r = (float(np.exp(ab[0])) * render + ab[1] - gt_color)[:, mask]
    h = 1e-8
    assert float(r.abs().min()) > 100 * h * (1 + float(render.abs().max()))
    fd = central(lambda e: mapping_statement(inputs, e)[0][0], ab, h)
    assert np.abs(fd - gE.numpy()).max() <= 1e-6 * np.abs(gE.numpy()).max(), (fd, gE)
    # the depth and normal terms do not see the exposure
    p0, _, gD0, gN0, _ = mapping_statement(inputs, (0.0, 0.0))
    assert parts[2:6] == p0[2:6] and torch.equal(gD, gD0) and torch.equal(gN, gN0)
    # dL/dC = e^a times the unexposed statement's sign pattern at the exposed residual
    assert float((gC - float(np.exp(ab[0])) * 0.8 / (3 * float(mask.sum())) * torch.sign(float(np.exp(ab[0])) * render + ab[1]
                                                                                         - gt_color) * mask).abs().max()) <= 1e-15


def ssim_inputs(C_, H, W, seed=4):
    gen = torch.Generator().manual_seed(seed)
    x = torch.rand(C_, H, W, generator=gen, dtype=torch.float64)
    y = (0.7 * x + 0.3 * torch.rand(C_, H, W, generator=gen, dtype=torch.float64)).clamp(0, 1)
    return x, y


def ssim_statement(x, y, ab):
    """1 - ssim(e^a x + b, y) in float64 (loss._ssim_term) and its autograd gradients w.r.t. x and (a, b)."""
    from rtg_slam_b200.loss import _ssim_term
    x = x.detach().clone().requires_grad_(True)
    e = torch.tensor(ab, dtype=torch.float64, requires_grad=True)
    v = _ssim_term(torch.exp(e[0]) * x + e[1], y)
    gx, ge = torch.autograd.grad(v, (x, e))
    return float(v.detach()), gx, ge


@pytest.mark.parametrize("shape", [(3, 37, 53), (1, 16, 16), (2, 5, 40)])
@pytest.mark.parametrize("ab", EXPOSURES)
def test_ssim_statement_under_an_exposure_matches_central_differences(ab, shape):
    x, y = ssim_inputs(*shape)
    v, gx, ge = ssim_statement(x, y, ab)
    h = 1e-6
    f = lambda e: ssim_statement(x, y, e)[0]
    fd = central(f, ab, h)
    assert np.abs(fd - ge.numpy()).max() <= 1e-6 * np.abs(ge.numpy()).max() + 1e-10, (fd, ge)
    # dL/dx = e^a dL/dx^: the gradient w.r.t. the exposed image, scaled
    from rtg_slam_b200.loss import _ssim_term
    xh = (float(np.exp(ab[0])) * x + ab[1]).requires_grad_(True)
    (gxh,) = torch.autograd.grad(_ssim_term(xh, y), (xh,))
    assert float((gx - float(np.exp(ab[0])) * gxh).abs().max()) <= 1e-12 * float(gx.abs().max())
    assert abs(float((gxh * float(np.exp(ab[0])) * x).sum()) - float(ge[0])) <= 1e-10 * abs(float(ge[0])) + 1e-15
    assert abs(float(gxh.sum()) - float(ge[1])) <= 1e-10 * abs(float(ge[1])) + 1e-15
    # (0, 0) is the plain term
    if ab == (0.0, 0.0):
        assert v == float(_ssim_term(x, y))


def test_loss_mapping_exposure_validates_before_touching_cuda():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    ok = C.c_void_p(256)
    names = ("render", "depth", "normal", "depth_index", "gt_color", "gt_depth", "gt_normal", "mask", "exposure", "dL_dcolor",
             "dL_ddepth", "dL_dnormal", "dL_dexposure", "loss_out", "ws")

    def call(H=16, W=16, normal_weight=0.1, **over):
        p = {k: ok for k in names}
        p.update(over)
        return L.rtg_loss_mapping_exposure(p["render"], p["depth"], p["normal"], p["depth_index"], p["gt_color"], p["gt_depth"],
                                           p["gt_normal"], p["mask"], H, W, 0, 0.8, 1.0, normal_weight, 0.1, p["exposure"],
                                           p["dL_dcolor"], p["dL_ddepth"], p["dL_dnormal"], p["dL_dexposure"], p["loss_out"], p["ws"],
                                           None)
    for kw in (dict(H=0), dict(W=-1)):
        assert call(**kw) == -1 and b"H and W must be >= 1" in L.rtg_last_error(), kw
    for k in ("render", "depth", "depth_index", "gt_color", "gt_depth", "dL_dcolor", "dL_ddepth", "loss_out", "ws"):
        assert call(**{k: None}) == -1 and b"NULL pointer" in L.rtg_last_error(), k
    assert call(mask=None, ws=C.c_void_p(260)) == -1 and b"8-byte aligned" in L.rtg_last_error()
    for k in ("exposure", "dL_dexposure"):
        assert call(**{k: None}) == -1 and b"NULL exposure" in L.rtg_last_error(), k
    for k in ("normal", "gt_normal", "dL_dnormal"):
        assert call(**{k: None}) == -1 and b"normal_weight > 0 needs" in L.rtg_last_error(), k
    assert b"rtg_loss_mapping_exposure" in L.rtg_last_error()


def test_ssim_loss_exposure_validates_before_touching_cuda():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    ok = C.c_void_p(256)

    def call(Cn=3, H=16, W=16, **over):
        p = {k: ok for k in ("img1", "img2", "exposure", "dL_dimg1", "dL_dexposure", "loss_out", "ws")}
        p.update(over)
        return L.rtg_ssim_loss_exposure(p["img1"], p["img2"], Cn, H, W, p["exposure"], p["dL_dimg1"], p["dL_dexposure"], p["loss_out"],
                                        p["ws"], None)
    for k in ("img1", "img2", "exposure", "loss_out", "ws"):
        assert call(**{k: None}) == -1 and b"NULL pointer" in L.rtg_last_error(), k
    for kw in (dict(Cn=0), dict(Cn=65536), dict(H=0), dict(W=-3), dict(H=65535 * 16 + 1)):
        assert call(**kw) == -1 and b"bad size" in L.rtg_last_error(), kw
    assert call(dL_dimg1=None, dL_dexposure=None, ws=C.c_void_p(260)) == -1 and b"8-byte aligned" in L.rtg_last_error()
    assert b"rtg_ssim_loss_exposure" in L.rtg_last_error()


def test_ssim_exposure_workspace_is_monotone_and_holds_the_plain_one():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    for bad in ((0, 16, 16), (3, 0, 16), (3, 16, -1)):
        assert L.rtg_ssim_exposure_workspace_bytes(*bad) == 0
    base = (3, 37, 53)
    for axis in range(3):
        prev = 0
        for v in (1, 16, 17, 100, 680):
            shape = list(base)
            shape[axis] = v
            n = L.rtg_ssim_exposure_workspace_bytes(*shape)
            tiles = shape[0] * ((shape[1] + 15) // 16) * ((shape[2] + 15) // 16)
            assert n >= L.rtg_ssim_workspace_bytes(*shape) + 2 * 8 * tiles and n >= prev, (shape, n, prev)
            prev = n


def test_keyframe_table_rejects_bad_hyper_parameters():
    from rtg_slam_b200.keyframes import KeyframeTable
    for kw in (dict(lr_rot=-1.0), dict(lr_exposure=-1e-3), dict(betas=(1.0, 0.999)), dict(eps=-1.0)):
        args = dict(lr_rot=1e-3, lr_trans=1e-3, lr_exposure=1e-2)
        args.update(kw)
        with pytest.raises(ValueError):
            KeyframeTable(**args)
    assert len(KeyframeTable(1e-3, 1e-3, 1e-2)) == 0
