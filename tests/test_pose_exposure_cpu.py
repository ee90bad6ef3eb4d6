"""CPU tests of exposure estimation in the pose refiners: a float64 statement of the eight-unknown Gauss-Newton step
(pose twist and the frame's exposure (a, b), C^ ~ e^a C + b; reused by the GPU tests), pinned against autograd and, without
the exposure columns, against the six-unknown statement; a float64 statement of the three frame losses (L1, L1 under an
exposure, mapping with the cosine normal term; reused by the GPU tests) against autograd and the eager expressions of the
mapping loss; the invariance of (a, b) under the pyramid's block mean; host validation of rtg_splat_pose_gn_step_exposure
and rtg_loss_l1_exposure and the RtgPoseExposure layout."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_pose_gn_cpu import gn_step, normal_equations, random_problem, se3_exp_closed
from test_pose_gn_pyramid_cpu import downsample_statement, huber, huber_weight
from test_pose_refine_cpu import POSES


# ------------------------------------------------------------------------------------------- the eight-unknown statement
def exposure_normal_equations(Jc, Cr, gt, sel_c, Jd, rd, sel_d, color_weight, depth_weight, ab, deltas=None):
    """H (8,8), g (8), (E, E_colour, E_depth), N_c, N_d of the objective over x = (xi, a, b) with the colour residual
    r = e^a C + b - C^ and the Jacobian row (e^a dC/dxi, e^a C, 1); the depth rows have zeros in columns 6, 7.
    Jc (6, 3, n) = dC/dxi, Cr, gt (3, n), Jd (6, n), rd (n), sel_* boolean (n,); deltas None (squared residuals) or the
    Huber thresholds (colour, depth): weights 1 or delta / |r| per residual. Float64."""
    a, b = float(ab[0]), float(ab[1])
    nc, nd = 3.0 * float(sel_c.sum()), float(sel_d.sum())
    wc = color_weight / nc if nc > 0 else 0.0
    wd = depth_weight / nd if nd > 0 else 0.0
    Jc, Cr, gt = Jc[..., sel_c], Cr[:, sel_c], gt[:, sel_c]
    Jd, rd = Jd[:, sel_d], rd[sel_d]
    ea = float(np.exp(a))
    rc = ea * Cr + b - gt
    J8 = torch.cat([ea * Jc, (ea * Cr)[None], torch.ones_like(Cr)[None]])           # (8, 3, n)
    if deltas is None:
        uc, ud = torch.ones_like(rc), torch.ones_like(rd)
        ec, ed = 0.5 * wc * float((rc * rc).sum()), 0.5 * wd * float((rd * rd).sum())
    else:
        uc, ud = huber_weight(rc, deltas[0]), huber_weight(rd, deltas[1])
        ec, ed = wc * float(huber(rc, deltas[0]).sum()), wd * float(huber(rd, deltas[1]).sum())
    H = wc * torch.einsum("acn,bcn,cn->ab", J8, J8, uc)
    g = wc * torch.einsum("acn,cn->a", J8, uc * rc)
    H[:6, :6] += wd * (Jd * ud) @ Jd.t()
    g[:6] += wd * Jd @ (ud * rd)
    return H, g, (ec + ed, ec, ed), nc, nd


def exposure_gn_step(H, g, damping, w2c, ab, exposed=True):
    """The device step from H and g: damping * trace(H[0:6, 0:6]) on the six pose diagonals, the exposure diagonals scaled
    by 1 + damping, Cholesky solve, closed-form exponential, a += x_6, b += x_7. `exposed` False (no colour term): the
    6x6 pose system alone, (a, b) kept. Returns (new W2C, new (a, b), x) or (w2c, ab, None) when not positive definite."""
    ab = torch.as_tensor(ab, dtype=torch.float64)
    if not exposed:
        new, xi = gn_step(H[:6, :6], g[:6], damping, w2c)
        return new, ab, xi
    A = H.clone()
    A[:6, :6] += damping * torch.trace(H[:6, :6]) * torch.eye(6, dtype=H.dtype)
    A[6, 6] *= 1 + damping
    A[7, 7] *= 1 + damping
    L, info = torch.linalg.cholesky_ex(A)
    if int(info) != 0:
        return w2c, ab, None
    x = torch.cholesky_solve(-g[:, None], L)[:, 0]
    return se3_exp_closed(x[:6]) @ w2c, ab + x[6:], x


def exposure_problem(seed, n=500):
    Jc, rc, sel_c, Jd, rd, sel_d = random_problem(seed, n)
    gen = torch.Generator().manual_seed(seed + 100)
    Cr = torch.rand(3, n, generator=gen, dtype=torch.float64)
    return Jc, Cr, Cr - 0.2 * rc, sel_c, Jd, rd, sel_d       # gt = C - 0.2 r: residuals of either sign at (0, 0)


@pytest.mark.parametrize("robust", [False, True])
@pytest.mark.parametrize("ab", [(0.0, 0.0), (0.2, 0.05), (-0.25, -0.03)])
def test_gradient_is_the_autograd_gradient(ab, robust):
    """g is the gradient of E over (xi, a, b) with the render linearised through J, C(xi) = C + J xi, at xi = 0."""
    Jc, Cr, gt, sel_c, Jd, rd, sel_d = exposure_problem(3)
    deltas = None
    if robust:
        r0 = float(np.exp(ab[0])) * Cr[:, sel_c] + ab[1] - gt[:, sel_c]
        deltas = (float(r0.abs().quantile(0.7)), float(rd[sel_d].abs().quantile(0.7)))
    H, g, (E, ec, ed), nc, nd = exposure_normal_equations(Jc, Cr, gt, sel_c, Jd, rd, sel_d, 0.8, 1.0, ab, deltas)
    x = torch.zeros(6, dtype=torch.float64, requires_grad=True)
    e = torch.tensor(ab, dtype=torch.float64, requires_grad=True)
    rcl = torch.exp(e[0]) * (Cr[:, sel_c] + torch.einsum("a,acn->cn", x, Jc[..., sel_c])) + e[1] - gt[:, sel_c]
    rdl = rd[sel_d] + x @ Jd[:, sel_d]
    if robust:
        El = 0.8 / nc * huber(rcl, deltas[0]).sum() + 1.0 / nd * huber(rdl, deltas[1]).sum()
        assert 0.2 < float((rcl.detach().abs() > deltas[0]).double().mean()) < 0.4
    else:
        El = 0.5 * (0.8 / nc * (rcl ** 2).sum() + 1.0 / nd * (rdl ** 2).sum())
    gx, ge = torch.autograd.grad(El, (x, e))
    gl = torch.cat([gx, ge])
    assert abs(float(El.detach()) - E) <= 1e-12 * abs(E) and abs(ec + ed - E) <= 1e-15 * abs(E)
    assert float((gl - g).abs().max()) <= 1e-12 * float(g.abs().max())
    assert torch.allclose(H, H.t()) and float(torch.linalg.eigvalsh(H).min()) > 0
    assert float(H[6:, :6].abs().max()) > 0
    if not robust:
        assert float(H[7, 7]) == pytest.approx(0.8)  # H_bb = color_weight


def test_without_the_exposure_columns_it_is_the_six_unknown_statement():
    Jc, Cr, gt, sel_c, Jd, rd, sel_d = exposure_problem(4)
    H8, g8, E8, nc8, nd8 = exposure_normal_equations(Jc, Cr, gt, sel_c, Jd, rd, sel_d, 0.8, 1.0, (0.0, 0.0))
    H, g, E, nc, nd = normal_equations(Jc, Cr - gt, sel_c, Jd, rd, sel_d, 0.8, 1.0)
    assert (nc8, nd8) == (nc, nd)
    assert float((H8[:6, :6] - H).abs().max()) <= 1e-12 * float(H.abs().max())
    assert float((g8[:6] - g).abs().max()) <= 1e-12 * float(g.abs().max())
    for p, q in zip(E8, E):
        assert abs(p - q) <= 1e-12 * abs(q)
    # the damping of the pose block is the six-unknown step's: with the exposure rows and columns cut, the same step
    w2c = POSES["rotated"]
    H6 = torch.zeros_like(H8)
    H6[:6, :6], H6[6, 6], H6[7, 7] = H8[:6, :6], 1.0, 1.0
    g6 = torch.cat([g8[:6], torch.zeros(2, dtype=torch.float64)])
    new8, ab, x = exposure_gn_step(H6, g6, 1e-4, w2c, (0.0, 0.0))
    new, xi = gn_step(H, g, 1e-4, w2c)
    assert float((x[:6] - xi).abs().max()) <= 1e-12 * float(xi.abs().max()) and float(x[6:].abs().max()) == 0
    assert float((new8 - new).abs().max()) <= 1e-12 and float(ab.abs().max()) == 0


def test_the_step_solves_the_damped_system_and_updates_the_exposure():
    Jc, Cr, gt, sel_c, Jd, rd, sel_d = exposure_problem(5)
    ab0 = (0.1, -0.02)
    H, g, _, _, _ = exposure_normal_equations(Jc, Cr, gt, sel_c, Jd, rd, sel_d, 0.8, 1.0, ab0)
    w2c = POSES["rotated"]
    new, ab, x = exposure_gn_step(H, g, 1e-4, w2c, ab0)
    D = torch.zeros((8, 8), dtype=torch.float64)
    D[:6, :6] = 1e-4 * torch.trace(H[:6, :6]) * torch.eye(6, dtype=torch.float64)
    D[6, 6], D[7, 7] = 1e-4 * H[6, 6], 1e-4 * H[7, 7]
    x_ref = torch.linalg.solve(H + D, -g)
    assert float((x - x_ref).abs().max()) <= 1e-12 * float(x_ref.abs().max())
    from test_pose_refine_cpu import hat
    ref = torch.matrix_exp(hat(x_ref[:6])) @ w2c
    assert float((new - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max()))
    assert float((ab - (torch.tensor(ab0, dtype=torch.float64) + x_ref[6:])).abs().max()) <= 1e-13
    # the exposure diagonals do not see the pose trace: H_bb = color_weight stays of order one in the damped system
    assert float(H[7, 7]) == pytest.approx(0.8) and float(torch.trace(H[:6, :6])) > float(H[7, 7])


def test_no_colour_term_leaves_the_exposure():
    """N_c = 0 (or color_weight = 0): the exposure columns are empty, the pose system is solved alone."""
    Jc, Cr, gt, sel_c, Jd, rd, sel_d = exposure_problem(6)
    w2c = POSES["rotated"]
    for kw in (dict(sel=torch.zeros_like(sel_c), cw=0.8), dict(sel=sel_c, cw=0.0)):
        H, g, (E, ec, ed), nc, nd = exposure_normal_equations(Jc, Cr, gt, kw["sel"], Jd, rd, sel_d, kw["cw"], 1.0, (0.2, 0.05))
        assert ec == 0.0 and float(H[6:].abs().max()) == 0 and float(g[6:].abs().max()) == 0
        assert exposure_gn_step(H, g, 1e-4, w2c, (0.2, 0.05))[2] is None        # the 8x8 system is singular
        new, ab, xi = exposure_gn_step(H, g, 1e-4, w2c, (0.2, 0.05), exposed=False)
        H6, g6, _, _, _ = normal_equations(Jc, Cr - gt, kw["sel"], Jd, rd, sel_d, kw["cw"], 1.0)
        want, xi6 = gn_step(H6, g6, 1e-4, w2c)
        assert xi is not None and torch.equal(ab, torch.tensor([0.2, 0.05], dtype=torch.float64))
        assert float((new - want).abs().max()) <= 1e-12


# -------------------------------------------------------------------------------------------- the frame loss statement
def loss_statement(render, depth, hit, gt_color, gt_depth, mask, color_weight, depth_weight, depth_error_max, ab=(0.0, 0.0),
                   normal=None, gt_normal=None, normal_weight=0.0, depth_near=None):
    """The three frame losses in float64: rtg_loss_l1 (ab = (0, 0), no normal), rtg_loss_l1_exposure (ab) and
    rtg_loss_mapping (normal, gt_normal and normal_weight > 0: the cosine normal term). Returns parts [total, colour,
    depth, n_depth, normal, n_normal, 0, 0] (a list of floats), dL/dC (3, n), dL/ddepth (n), dL/dnormal (3, n) or None,
    dL/d(a, b) (2).
    render, gt_color, normal, gt_normal (3, n); depth, gt_depth (n); hit (n) int; mask (n) bool. Colour: mean |e^a C + b -
    C^| over 3 x the masked pixels. Depth: mean |D - D^| over mask & hit != -1 & D^ > 0 & D - D^ < depth_error_max; the
    error test is `depth_near` (n) bool if given (the GPU tests pass the float32 comparison the kernel makes). Normal:
    mean (1 - cos) over mask & hit != -1 & gt_normal != (0, 0, 0), cos = x.y / (max(|x|, 1e-8) max(|y|, 1e-8))
    (F.cosine_similarity). Every mean over an empty set, and its gradient, is 0. The tensors may live on any device."""
    a, b = float(ab[0]), float(ab[1])
    ea = float(np.exp(a))
    f64 = dict(dtype=torch.float64, device=render.device)
    r = torch.where(mask[None], ea * render + b - gt_color, torch.zeros_like(render))
    n = float(mask.sum())
    e = depth - gt_depth
    sel_d = mask & (hit != -1) & (gt_depth > 0) & ((e < depth_error_max) if depth_near is None else depth_near)
    nd = float(sel_d.sum())
    gcs = color_weight / (3 * n) if n > 0 else 0.0
    gds = depth_weight / nd if nd > 0 else 0.0
    cl = float(r.abs().sum()) / (3 * n) if n > 0 else 0.0
    dl = float(e[sel_d].abs().sum()) / nd if nd > 0 else 0.0
    sg = torch.sign(r)
    nl, nn, gN = 0.0, 0.0, None
    if normal is not None and normal_weight > 0:
        sel_n = mask & (hit != -1) & (gt_normal != 0).any(0)
        nn = float(sel_n.sum())
        xl, yl = normal.norm(dim=0), gt_normal.norm(dim=0)
        nx, ny = xl.clamp_min(1e-8), yl.clamp_min(1e-8)
        cos = (normal * gt_normal).sum(0) / (nx * ny)
        nl = float((1 - cos)[sel_n].sum()) / nn if nn > 0 else 0.0
        gns = normal_weight / nn if nn > 0 else 0.0
        # d cos / dx = y / (nx ny) - cos x / |x|^2 where |x| > 1e-8 (below, nx is the constant 1e-8)
        dcos = gt_normal / (nx * ny) - torch.where(xl > 1e-8, cos / (nx * nx), torch.zeros_like(cos)) * normal
        gN = -gns * dcos * sel_n
    total = color_weight * cl + depth_weight * dl + (normal_weight * nl if gN is not None else 0.0)
    return ([total, cl, dl, nd, nl, nn, 0.0, 0.0], gcs * ea * sg, gds * torch.sign(e) * sel_d, gN,
            torch.tensor([gcs * float((sg * ea * render).sum()), gcs * float(sg.sum())], **f64))


@pytest.mark.parametrize("ab", [(0.0, 0.0), (0.2, 0.05), (-0.25, -0.03)])
def test_l1_exposure_statement_matches_autograd(ab):
    gen = torch.Generator().manual_seed(9)
    n = 400
    render = torch.rand(3, n, generator=gen, dtype=torch.float64).requires_grad_(True)
    gt_color = torch.rand(3, n, generator=gen, dtype=torch.float64)
    depth = (1 + torch.rand(n, generator=gen, dtype=torch.float64)).requires_grad_(True)
    gt_depth = depth.detach() + 0.08 * torch.randn(n, generator=gen, dtype=torch.float64)
    gt_depth[::17] = 0.0
    hit = torch.where(torch.rand(n, generator=gen) < 0.9, 1, -1)
    mask = torch.rand(n, generator=gen) < 0.8
    (loss, cl, dl, nd, *_), gC, gD, _, gE = loss_statement(render.detach(), depth.detach(), hit, gt_color, gt_depth, mask, 0.8, 1.0,
                                                           0.1, ab)
    e = torch.tensor(ab, dtype=torch.float64, requires_grad=True)
    sel_d = mask & (hit != -1) & (gt_depth > 0) & ((depth.detach() - gt_depth) < 0.1)
    L = (0.8 * (torch.exp(e[0]) * render + e[1] - gt_color)[:, mask].abs().mean() + 1.0 * (depth - gt_depth)[sel_d].abs().mean())
    aC, aD, aE = torch.autograd.grad(L, (render, depth, e))
    assert 0 < nd < n and abs(float(L.detach()) - loss) <= 1e-12 * loss
    assert float((aC - gC).abs().max()) <= 1e-15 and float((aD - gD).abs().max()) <= 1e-15
    assert float((aE - gE).abs().max()) <= 1e-12 * float(aE.abs().max())


def mapping_frame(H, W, gen, dtype=torch.float64):
    """A frame for the mapping loss as the loss tests build it: about half the depths within 0.1 of gt, 10 % of gt depths
    0, 15 % of gt normals the zero vector and some with one or two zero components; render normals of length 0.5 - 1.5.
    Returns render (3,H,W), depth (1,H,W), normal (3,H,W), depth_index (1,H,W) int32, gt_color (H,W,3), gt_depth (H,W,1),
    gt_normal (H,W,3). `gen` is a torch.Generator; the tensors live on its device."""
    import torch.nn.functional as F
    kw = dict(generator=gen, device=gen.device)
    u = lambda *s: torch.rand(*s, **kw)
    render = u(3, H, W).to(dtype)
    depth = (u(1, H, W) * 3).to(dtype)
    normal = (F.normalize(torch.randn(3, H, W, **kw), dim=0) * (0.5 + u(1, H, W))).to(dtype)
    depth_index = torch.randint(-1, 50, (1, H, W), dtype=torch.int32, **kw)
    gt_color = u(H, W, 3).to(dtype)
    near = depth.permute(1, 2, 0) + 0.05 * torch.randn(H, W, 1, **kw).to(dtype)
    gt_depth = torch.where(u(H, W, 1) < 0.5, near, (u(H, W, 1) * 3).to(dtype))
    gt_depth[u(H, W, 1) < 0.1] = 0
    gt_normal = F.normalize(torch.randn(H, W, 3, **kw), dim=-1).to(dtype)
    k = u(H, W)
    gt_normal[k < 0.15] = 0
    gt_normal[(k >= 0.15) & (k < 0.2), 0] = 0                                  # one zero component
    gt_normal[(k >= 0.2) & (k < 0.25), 1:] = 0                                 # two zero components
    return render, depth, normal, depth_index, gt_color, gt_depth, gt_normal


@pytest.mark.parametrize("use_mask", [False, True])
def test_loss_statement_is_the_mapping_loss_expressions(use_mask):
    """The statement with the normal term against the eager expressions of Mapping.loss_update (mapper.py:402-451), as
    test_mapping_loss_with_normal_and_ssim_terms writes them, differentiated by autograd in float64."""
    import torch.nn.functional as F
    H, W = 23, 31
    gen = torch.Generator().manual_seed(11)
    render, depth, normal, depth_index, gt_color, gt_depth, gt_normal = mapping_frame(H, W, gen)
    mask = (torch.rand(H, W, generator=gen) < 0.6) if use_mask else None
    for t in (render, depth, normal):
        t.requires_grad_(True)
    w = dict(color_weight=0.8, depth_weight=1.0, normal_weight=0.1)
    image, d, nrm, di = render.permute(1, 2, 0), depth.permute(1, 2, 0), normal.permute(1, 2, 0), depth_index.permute(1, 2, 0)
    rm = torch.ones(H, W, dtype=torch.bool) if mask is None else mask
    color_loss = torch.abs(image[rm] - gt_color[rm]).mean()
    err = d - gt_depth
    valid = (di != -1).squeeze() & (gt_depth > 0).squeeze() & (err < 0.1).squeeze() & rm
    depth_loss = torch.abs(err[valid]).mean()
    cos_dist = 1 - F.cosine_similarity(nrm, gt_normal, dim=-1)
    vn = rm & (di != -1).squeeze() & (~(gt_normal == 0).all(dim=-1))
    normal_loss = cos_dist[vn].mean()
    ref = w["depth_weight"] * depth_loss + w["normal_weight"] * normal_loss + w["color_weight"] * color_loss
    aC, aD, aN = torch.autograd.grad(ref, (render, depth, normal))
    n = H * W
    parts, gC, gD, gN, gE = loss_statement(render.detach().reshape(3, n), depth.detach().reshape(n), depth_index.reshape(n),
                                           gt_color.permute(2, 0, 1).reshape(3, n), gt_depth.reshape(n), rm.reshape(n), w["color_weight"],
                                           w["depth_weight"], 0.1, normal=normal.detach().reshape(3, n),
                                           gt_normal=gt_normal.permute(2, 0, 1).reshape(3, n), normal_weight=w["normal_weight"])
    # the frame has every kind of pixel: a gt normal with one or two zero components takes part in the normal term
    partial = (gt_normal == 0).any(-1) & ~(gt_normal == 0).all(-1)
    assert 0 < parts[3] < n and 0 < parts[5] < n and int((vn & partial).sum()) > 0 and int((~vn & rm).sum()) > 0
    assert parts[5] == int(vn.sum()) and parts[3] == int(valid.sum()) and parts[6:] == [0.0, 0.0]
    for got, want in zip(parts[:3] + parts[4:5], (ref, color_loss, depth_loss, normal_loss)):
        want = float(want.detach())
        assert abs(got - want) <= 1e-13 * abs(want), (got, want)
    for got, want in ((gC, aC), (gD, aD), (gN, aN)):
        assert float((got.reshape(want.shape) - want).abs().max()) <= 1e-14 * float(want.abs().max())
    # without the normal weight the statement is the L1 one: parts 4 and 5 are 0 and there is no normal gradient
    p0, c0, d0, n0, _ = loss_statement(render.detach().reshape(3, n), depth.detach().reshape(n), depth_index.reshape(n),
                                       gt_color.permute(2, 0, 1).reshape(3, n), gt_depth.reshape(n), rm.reshape(n), 0.8, 1.0, 0.1,
                                       normal=normal.detach().reshape(3, n), gt_normal=gt_normal.permute(2, 0, 1).reshape(3, n))
    assert n0 is None and p0[4:6] == [0.0, 0.0] and p0[1:4] == parts[1:4] and torch.equal(c0, gC) and torch.equal(d0, gD)


# ------------------------------------------------------------------------------------------------------- the pyramid
@pytest.mark.parametrize("s", [2, 4])
def test_the_block_mean_keeps_the_exposure(s):
    """downsample(e^a C + b) = e^a downsample(C) + b: the exposure of a frame is the exposure of each of its levels."""
    rng = np.random.default_rng(3)
    H, W = 37, 50
    color = rng.uniform(size=(3, H, W)).astype(np.float32)
    depth = rng.uniform(0.5, 3.0, size=(H, W)).astype(np.float32)
    for a, b in ((0.2, 0.05), (-0.25, -0.03)):
        seen = (np.float32(np.exp(a)) * color + np.float32(b)).astype(np.float32)
        lhs = downsample_statement(seen, depth, s)[0]
        rhs = np.float32(np.exp(a)) * downsample_statement(color, depth, s)[0] + np.float32(b)
        assert np.abs(lhs - rhs).max() <= 1e-6


# ------------------------------------------------------------------------------------------------- host validation
def test_exposure_struct_layout_and_scratch_bytes():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    assert C.sizeof(_lib.RtgPoseExposure) == 8 and _lib.RtgPoseExposure.ab.offset == 0
    tiles = 3 * 4
    assert L.rtg_splat_pose_gn_exposure_scratch_bytes(1000, 48, 64) == ((1000 * 192 + 255) // 256) * 256 + tiles * 75 * 8
    assert L.rtg_splat_pose_gn_exposure_scratch_bytes(-1, 48, 64) == 0 and L.rtg_splat_pose_gn_exposure_scratch_bytes(10, 0, 64) == 0
    prev = 0
    for P, H, W in ((10, 16, 16), (10, 48, 64), (1000, 48, 64), (1000, 480, 640), (100000, 680, 1200)):
        n = L.rtg_splat_pose_gn_exposure_scratch_bytes(P, H, W)
        assert n > prev and n >= L.rtg_splat_pose_gn_scratch_bytes(P, H, W)
        prev = n
    assert L.rtg_loss_l1_exposure_workspace_bytes() >= L.rtg_loss_workspace_bytes()


def test_pose_gn_step_exposure_validates_before_touching_cuda():
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    ok = C.c_void_p(256)
    view = _lib.RtgSplatView()
    view.image_height, view.image_width, view.sh_degree = 48, 64, 3
    view.viewmatrix = view.projmatrix = view.campos = view.bg = 256  # never dereferenced: validation fails first

    def state(**over):
        s = _lib.RtgPoseGN()
        for k in ("pose", "projection", "viewmatrix", "projmatrix", "campos", "render", "depth", "hit_depth", "gt_color", "gt_depth",
                  "scratch", "report"):
            setattr(s, k, 256)
        s.color_weight, s.depth_weight, s.depth_error_max, s.damping = 0.8, 1.0, 0.1, 1e-4
        for k, v in over.items():
            setattr(s, k, v)
        return s

    def robust(kernel=1, dc=0.1, dd=0.05):
        r = _lib.RtgPoseRobust()
        r.kernel, r.color_delta, r.depth_delta = kernel, dc, dd
        return r

    def exposure(ab=256):
        e = _lib.RtgPoseExposure()
        e.ab = ab
        return e

    def call(st=state(), r=robust(), e=exposure(), P=4, v=C.byref(view)):
        ref = lambda x: None if x is None else C.byref(x)
        return L.rtg_splat_pose_gn_step_exposure(v, P, 16, ok, ok, None, ok, ok, None, ok, ok, ok, 1024, ok, ref(st), ref(r), ref(e),
                                                 None)
    assert call(st=None) == -1 and b"state is NULL" in L.rtg_last_error()
    assert call(r=None) == -1 and b"robust is NULL" in L.rtg_last_error()
    assert call(e=None) == -1 and b"exposure is NULL" in L.rtg_last_error()
    assert call(e=exposure(None)) == -1 and b"exposure ab is NULL" in L.rtg_last_error()
    assert call(e=exposure(260)) == -1 and b"8-byte aligned" in L.rtg_last_error()
    for k in (-1, 2, 7):
        assert call(r=robust(kernel=k)) == -1 and b"unknown robust kernel" in L.rtg_last_error(), k
    for dc, dd in ((0.0, 0.05), (float("nan"), 0.05), (0.1, -1.0), (0.1, float("inf"))):
        assert call(r=robust(dc=dc, dd=dd)) == -1 and b"positive and finite" in L.rtg_last_error(), (dc, dd)
    # everything rtg_splat_pose_gn_step rejects; RTG_ROBUST_NONE ignores the deltas
    assert call(v=None) == -1 and b"view is NULL" in L.rtg_last_error()
    assert call(P=0) == -1 and b"P must be >= 1" in L.rtg_last_error()
    assert call(r=robust(kernel=0, dc=float("nan"), dd=-1.0), P=0) == -1 and b"P must be >= 1" in L.rtg_last_error()
    for k in ("hit_depth", "scratch"):
        assert call(st=state(**{k: None})) == -1 and b"NULL pointer" in L.rtg_last_error(), k
    for k in ("pose", "projection", "viewmatrix", "projmatrix", "campos", "report"):
        assert call(st=state(**{k: None})) == -1 and b"NULL pose / projection" in L.rtg_last_error(), k
    for k in ("render", "depth", "gt_color", "gt_depth"):
        assert call(st=state(**{k: None})) == -1 and b"NULL render" in L.rtg_last_error(), k
    assert call(st=state(pose=260)) == -1 and b"8-byte aligned" in L.rtg_last_error()
    for k in ("damping", "color_weight", "depth_weight"):
        assert call(st=state(**{k: -1.0})) == -1 and b">= 0" in L.rtg_last_error(), k
    assert b"rtg_splat_pose_gn_step_exposure" in L.rtg_last_error()


def test_loss_l1_exposure_validates_before_touching_cuda():
    """rtg_loss_l1_exposure, rtg_loss_l1 and rtg_loss_mapping share one host validation, each with its own extra rule."""
    from rtg_slam_b200 import _lib
    L = _lib.lib()
    ok = C.c_void_p(256)
    names = ("render", "depth", "normal", "depth_index", "gt_color", "gt_depth", "gt_normal", "mask", "exposure", "dL_dcolor",
             "dL_ddepth", "dL_dnormal", "dL_dexposure", "loss_out", "ws")

    def args(H, W, over):
        p = {k: ok for k in names}
        p.update(over)
        return p, H, W

    def exposure(H=16, W=16, **over):
        p, H, W = args(H, W, over)
        return L.rtg_loss_l1_exposure(p["render"], p["depth"], p["depth_index"], p["gt_color"], p["gt_depth"], p["mask"], H, W, 0,
                                      0.8, 1.0, 0.1, p["exposure"], p["dL_dcolor"], p["dL_ddepth"], p["dL_dexposure"], p["loss_out"],
                                      p["ws"], None)

    def l1(H=16, W=16, **over):
        p, H, W = args(H, W, over)
        return L.rtg_loss_l1(p["render"], p["depth"], p["depth_index"], p["gt_color"], p["gt_depth"], p["mask"], H, W, 0, 0.8, 1.0,
                             0.1, p["dL_dcolor"], p["dL_ddepth"], p["loss_out"], p["ws"], None)

    def mapping(H=16, W=16, normal_weight=0.1, **over):
        p, H, W = args(H, W, over)
        return L.rtg_loss_mapping(p["render"], p["depth"], p["normal"], p["depth_index"], p["gt_color"], p["gt_depth"], p["gt_normal"],
                                  p["mask"], H, W, 0, 0.8, 1.0, normal_weight, 0.1, p["dL_dcolor"], p["dL_ddepth"], p["dL_dnormal"],
                                  p["loss_out"], p["ws"], None)

    for call, who in ((exposure, b"rtg_loss_l1_exposure"), (l1, b"rtg_loss_l1:"), (mapping, b"rtg_loss_mapping")):
        for kw in (dict(H=0), dict(W=-1)):
            assert call(**kw) == -1 and b"H and W must be >= 1" in L.rtg_last_error(), (who, kw)
        for k in ("render", "depth", "depth_index", "gt_color", "gt_depth", "dL_dcolor", "dL_ddepth", "loss_out", "ws"):
            assert call(**{k: None}) == -1 and b"NULL pointer" in L.rtg_last_error(), (who, k)
        assert call(mask=None, ws=C.c_void_p(260)) == -1 and b"8-byte aligned" in L.rtg_last_error(), who
        assert who in L.rtg_last_error()
    for k in ("exposure", "dL_dexposure"):
        assert exposure(**{k: None}) == -1 and b"NULL exposure" in L.rtg_last_error(), k
    for k in ("normal", "gt_normal", "dL_dnormal"):
        assert mapping(**{k: None}) == -1 and b"normal_weight > 0 needs" in L.rtg_last_error(), k


def test_refiners_reject_a_malformed_exposure():
    from rtg_slam_b200.tracking import _exposure_pair, apply_exposure
    for bad in ((0.0,), (0.0, 0.0, 0.0), torch.zeros(3)):
        with pytest.raises(ValueError):
            _exposure_pair(bad, torch.device("cpu"), torch.float64)
    t = _exposure_pair(torch.tensor([0.2, 0.05]), torch.device("cpu"), torch.float64)
    assert t.dtype == torch.float64 and t.shape == (2,)
    img = torch.rand(3, 4, 5, dtype=torch.float64)
    want = float(np.exp(0.2)) * img + 0.05
    assert float((apply_exposure(img, (0.2, 0.05)) - want).abs().max()) <= 1e-15
    assert float((apply_exposure(img, torch.tensor([0.2, 0.05], dtype=torch.float64)) - want).abs().max()) <= 1e-15
