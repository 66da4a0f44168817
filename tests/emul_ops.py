"""TEST INFRASTRUCTURE: torch-CPU emulation of the libepb.so entry points with
the SAME signatures as epipolarpose_b200.ops, written directly from the
contracts in include/epb.h.  It lets the CPU test-suite exercise the host
logic (network plan, geometry/tap tables, weight packing, autograd wiring,
optimiser) without a GPU.  It is never imported by the product path."""
import numpy as np
import torch

from epipolarpose_b200._lib import ConvGeom, EPB_MAX_TAPS

launches = 0


def make_geom(N, Hi, Wi, Cin, Ho, Wo, Cout, Hp, Wp, os, ph, pw, is_, taps, Tw,
              in_relu=0, accumulate=0, precision=0):
    g = ConvGeom()
    g.N, g.Hi, g.Wi, g.Cin = N, Hi, Wi, Cin
    g.Ho, g.Wo, g.Cout = Ho, Wo, Cout
    g.Hp, g.Wp, g.os, g.ph, g.pw, g.is_ = Hp, Wp, os, ph, pw, is_
    g.T = len(taps)
    assert g.T <= EPB_MAX_TAPS
    for i, (dh, dw, wt) in enumerate(taps):
        g.dh[i], g.dw[i], g.wt[i] = dh, dw, wt
    g.Tw = Tw
    g.in_relu, g.accumulate, g.precision = in_relu, accumulate, precision
    return g


def _gather(g, x, t, in_scale, in_shift):
    """[N,Hp,Wp,Cin] = f(x[n, i*is+dh, j*is+dw, :]) with zero outside."""
    x = x.reshape(g.N, g.Hi, g.Wi, g.Cin)
    if in_scale is not None:
        x = x * in_scale + in_shift
        if g.in_relu:
            x = torch.relu(x)
    dh, dw = g.dh[t], g.dw[t]
    out = torch.zeros(g.N, g.Hp, g.Wp, g.Cin, dtype=x.dtype)
    ii = torch.arange(g.Hp) * g.is_ + dh
    jj = torch.arange(g.Wp) * g.is_ + dw
    vi = (ii >= 0) & (ii < g.Hi)
    vj = (jj >= 0) & (jj < g.Wi)
    if vi.any() and vj.any():
        sub = x[:, ii[vi]][:, :, jj[vj]]
        tmp = out[:, vi]
        tmp[:, :, vj] = sub
        out[:, vi] = tmp
    return out


def conv_fprop(g, x, w, out, in_scale=None, in_shift=None, bias=None, stats=None):
    W = w.reshape(g.Cout, g.Tw, g.Cin)
    acc = torch.zeros(g.N, g.Hp, g.Wp, g.Cout, dtype=torch.float32)
    for t in range(g.T):
        acc += _gather(g, x, t, in_scale, in_shift) @ W[:, g.wt[t], :].T
    if bias is not None:
        acc += bias
    o = out.view(g.N, g.Ho, g.Wo, g.Cout)
    sl = o[:, g.ph::g.os, g.pw::g.os][:, :g.Hp, :g.Wp]
    if g.accumulate:
        acc = acc + sl
    o[:, g.ph::g.os, g.pw::g.os][:, :g.Hp, :g.Wp] = acc
    if stats is not None:
        flat = acc.reshape(-1, g.Cout).double()
        stats[:g.Cout] += flat.sum(0)
        stats[g.Cout:] += (flat * flat).sum(0)


def conv_wgrad(g, x, dout, dw, in_scale=None, in_shift=None):
    DW = dw.view(g.Cout, g.Tw, g.Cin)
    d = dout.view(g.N, g.Ho, g.Wo, g.Cout)[:, g.ph::g.os, g.pw::g.os][:, :g.Hp, :g.Wp]
    d = d.reshape(-1, g.Cout)
    for t in range(g.T):
        a = _gather(g, x, t, in_scale, in_shift).reshape(-1, g.Cin)
        DW[:, g.wt[t], :] += d.T @ a


def pack_weight(src, dst, A, B, kh, kw, swap, ypad, unpack=0):
    T = kh * kw
    X, Y = (B, A) if swap else (A, B)
    if not unpack:
        s = src.reshape(A, B, T)
        p = s.permute(1, 2, 0) if swap else s.permute(0, 2, 1)   # [X][T][Y]
        d = dst.view(-1)[:X * T * ypad].view(X, T, ypad)
        d.zero_()
        d[:, :, :Y] = p
    else:
        p = src.view(-1)[:X * T * ypad].view(X, T, ypad)[:, :, :Y]
        d = dst.view(A, B, T)
        d.copy_(p.permute(2, 0, 1) if swap else p.permute(0, 2, 1))


class PackBatch:
    def __init__(self, jobs):
        self.jobs = list(jobs)


def pack_weight_batch(batch):
    for (src, dst, A, B, T, swap, ypad, unpack, xp) in batch.jobs:
        X, Y = (B, A) if swap else (A, B)
        if not unpack:
            s = src.reshape(A, B, T)
            p = s.permute(1, 2, 0) if swap else s.permute(0, 2, 1)   # [X][T][Y]
            d = torch.as_strided(dst.view(-1), (X, T, ypad), (xp, ypad, 1))
            d.zero_()
            d[:, :, :Y] = p
        else:
            p = torch.as_strided(src.view(-1), (X, T, ypad), (xp, ypad, 1))[:, :, :Y]
            d = dst.view(A, B, T)
            d.copy_(p.permute(2, 0, 1) if swap else p.permute(0, 2, 1))


def im2col(x, col, N, Hi, Wi, pitch, C, kh, kw, stride, pad, Ho, Wo, Kpad):
    xs = x.reshape(N, Hi, Wi, pitch)[..., :C]
    xp = torch.nn.functional.pad(xs, (0, 0, pad, pad, pad, pad))
    out = torch.zeros(N, Ho, Wo, Kpad)
    for r in range(kh):
        for s in range(kw):
            t = r * kw + s
            out[..., t * C:(t + 1) * C] = xp[:, r:r + stride * Ho:stride, s:s + stride * Wo:stride]
    col.view(N, Ho, Wo, Kpad).copy_(out)


def nchw_to_nhwc(src, dst, N, C, H, W, Cpad):
    d = dst.view(N, H, W, Cpad)
    d.zero_()
    d[..., :C] = src.view(N, C, H, W).permute(0, 2, 3, 1)


def nhwc_to_nchw(src, dst, N, C, H, W, Cpad):
    dst.view(N, C, H, W).copy_(src.view(N, H, W, Cpad)[..., :C].permute(0, 3, 1, 2))


def channel_stats(x, M, C, stats):
    f = x.reshape(M, C).double()
    stats[:C] += f.sum(0)
    stats[C:] += (f * f).sum(0)


def bn_finalize(stats, M, C, gamma, beta, eps, momentum, running_mean, running_var, scale, shift,
                mean, invstd):
    mu = stats[:C] / M
    var = (stats[C:] / M - mu * mu).clamp_min(0)
    inv = 1.0 / torch.sqrt(var + eps)
    scale.copy_((gamma.double() * inv).float())
    shift.copy_((beta.double() - mu * gamma.double() * inv).float())
    if mean is not None:
        mean.copy_(mu.float())
        invstd.copy_(inv.float())
    if running_mean is not None:
        running_mean.copy_(((1 - momentum) * running_mean.double() + momentum * mu).float())
        unb = var * (M / max(M - 1, 1))
        running_var.copy_(((1 - momentum) * running_var.double() + momentum * unb).float())


def bn_eval_affine(C, gamma, beta, running_mean, running_var, eps, scale, shift):
    s = gamma.double() / torch.sqrt(running_var.double() + float(torch.tensor(eps, dtype=torch.float32)))
    scale.copy_(s.float())
    shift.copy_((beta.double() - running_mean.double() * s).float())


def bn_act(x, scale, shift, r, rscale, rshift, relu, y, M, C):
    v = x.reshape(M, C)
    if scale is not None:
        v = v * scale + shift
    if r is not None:
        q = r.reshape(M, C)
        if rscale is not None:
            q = q * rscale + rshift
        v = v + q
    if relu:
        v = torch.relu(v)
    y.view(M, C).copy_(v)


def bn_relu_maxpool(x, scale, shift, y, argidx, N, H, W, C):
    a = torch.relu(x.view(N, H, W, C) * scale + shift).permute(0, 3, 1, 2)
    Ho, Wo = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
    pad = torch.nn.functional.pad(a, (1, 1, 1, 1), value=float("-inf"))
    best = torch.full((N, C, Ho, Wo), float("-inf"))
    bi = torch.zeros((N, C, Ho, Wo), dtype=torch.uint8)
    for kh in range(3):
        for kw in range(3):
            v = pad[:, :, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2]
            m = v > best
            best = torch.where(m, v, best)
            bi = torch.where(m, torch.full_like(bi, kh * 3 + kw), bi)
    y.view(N, Ho, Wo, C).copy_(best.permute(0, 2, 3, 1))
    argidx.view(N, Ho, Wo, C).copy_(bi.permute(0, 2, 3, 1))


def maxpool_bwd(dy, argidx, dx, N, H, W, C):
    Ho, Wo = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
    g = dy.view(N, Ho, Wo, C)
    k = argidx.view(N, Ho, Wo, C)
    pad = torch.zeros(N, H + 2, W + 2, C)
    for kh in range(3):
        for kw in range(3):
            sel = (k == kh * 3 + kw).float() * g
            pad[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] += sel
    dx.view(N, H, W, C).copy_(pad[:, 1:H + 1, 1:W + 1])


def _masked(dy, x, y_out, scale, shift, relu, M, C):
    g = dy.reshape(M, C)
    if y_out is not None:
        return g * (y_out.reshape(M, C) > 0).float()
    if relu:
        return g * ((x.reshape(M, C) * scale + shift) > 0).float()
    return g


def bn_bwd_reduce(dy, x, y_out, scale, shift, mean, invstd, relu, M, C, sums):
    g = _masked(dy, x, y_out, scale, shift, relu, M, C).double()
    xh = ((x.reshape(M, C) - mean) * invstd).double()
    sums[:C] += g.sum(0)
    sums[C:] += (g * xh).sum(0)


def bn_bwd_apply(dy, x, y_out, scale, shift, mean, invstd, gamma, relu, sums, M, C, dx, dgamma,
                 dbeta):
    g = _masked(dy, x, y_out, scale, shift, relu, M, C)
    xh = (x.reshape(M, C) - mean) * invstd
    k1 = (sums[:C] / M).float()
    k2 = (sums[C:] / M).float()
    dx.view(M, C).copy_(gamma * invstd * (g - k1 - xh * k2))
    if dgamma is not None:
        dgamma.copy_(sums[C:].float())
    if dbeta is not None:
        dbeta.copy_(sums[:C].float())


def add_masked(a, b, mask_src, dx, n):
    q = b.reshape(-1)
    if mask_src is not None:
        q = q * (mask_src.reshape(-1) > 0).float()
    dx.view(-1).copy_(a.reshape(-1) + q)


def avgpool(x, y, N, HW, C):
    y.view(N, C).copy_(x.reshape(N, HW, C).mean(1))


def avgpool_bwd(dy, dx, N, HW, C, accumulate):
    g = (dy.reshape(N, 1, C) / HW).expand(N, HW, C)
    d = dx.view(N, HW, C)
    if accumulate:
        d += g
    else:
        d.copy_(g)


def colsum(x, M, C, out):
    out.copy_(x.reshape(M, C).double().sum(0).float())


def _volume(logits, layout, N, J, D, H, W):
    if layout == 0:
        return logits.reshape(N, J, D, H, W)
    return logits.reshape(N, H, W, J, D).permute(0, 3, 4, 1, 2)


def softargmax_fwd(logits, layout, N, J, D, H, W, coords, lse):
    v = _volume(logits, layout, N, J, D, H, W).reshape(N * J, -1)
    m = v.max(1, keepdim=True).values
    e = torch.exp(v - m)
    s = e.sum(1, keepdim=True)
    p = (e / s).reshape(N * J, D, H, W)
    cx = (p.sum((1, 2)) * torch.arange(W)).sum(1) / W - 0.5
    cy = (p.sum((1, 3)) * torch.arange(H)).sum(1) / H - 0.5
    cz = (p.sum((2, 3)) * torch.arange(D)).sum(1) / D - 0.5
    coords.view(N * J, 3).copy_(torch.stack([cx, cy, cz], 1))
    lse.view(N * J, 2).copy_(torch.cat([m, 1.0 / s], 1))


def softargmax_bwd(logits, layout, N, J, D, H, W, coords, lse, dcoords, dlogits):
    v = _volume(logits, layout, N, J, D, H, W).reshape(N * J, D, H, W)
    l = lse.view(N * J, 2)
    p = torch.exp(v - l[:, 0, None, None, None]) * l[:, 1, None, None, None]
    g = dcoords.view(N * J, 3)
    c = coords.view(N * J, 3)
    s = (g[:, 0, None, None, None] * torch.arange(W)[None, None, None, :] / W
         + g[:, 1, None, None, None] * torch.arange(H)[None, None, :, None] / H
         + g[:, 2, None, None, None] * torch.arange(D)[None, :, None, None] / D)
    sbar = (g * (c + 0.5)).sum(1)
    d = (p * (s - sbar[:, None, None, None])).reshape(N, J, D, H, W)
    if layout == 0:
        dlogits.view(N, J, D, H, W).copy_(d)
    else:
        dlogits.view(N, H, W, J, D).copy_(d.permute(0, 3, 4, 1, 2))


def softargmax_bwd_split(logits, N, J, D, H, W, coords, lse, dcoords, dlogits16, sc, dbias):
    d = torch.empty(N, H, W, J * D)
    softargmax_bwd(logits, 1, N, J, D, H, W, coords, lse, dcoords, d)
    g = dcoords.view(N * J, 3).abs().sum(1)
    bound = float((lse.view(N * J, 2)[:, 1] * g).max())
    assert float(d.abs().max()) <= bound * (1 + 1e-5) + 1e-30, "logit gradient exceeds its bound"
    s = _pow2_scale(bound)
    sc[0], sc[1] = s, 1.0 / s
    _store_split(dlogits16, d.reshape(-1, J * D), s)
    if dbias is not None:
        dbias.copy_(d.reshape(-1, J * D).double().sum(0).float())


def heatmap_joint_loss(hm, target, hm_weight, R, HW, hm_scale, x, t, w, n, kind, div, jt_scale,
                       loss, dhm, dx):
    h = hm.reshape(R, HW).double()
    g = target.reshape(R, HW).double()
    wr = torch.ones(R, 1, dtype=torch.float64) if hm_weight is None else \
        hm_weight.reshape(R, 1).double()
    d = wr * (h - g)
    loss_hm = (d * d).mean()
    if dhm is not None:
        dhm.view(R, HW).copy_((2.0 * hm_scale * wr * d / (R * HW)).float())
    loss_jt = torch.zeros((), dtype=torch.float64)
    if n > 0:
        tmp = torch.empty(1)
        gx = torch.empty(n)
        jointloss(x, t, w, n, kind, 0, div, tmp, gx)
        loss_jt = tmp[0].double()
        if dx is not None:
            dx.view(-1).copy_(gx * jt_scale)
    loss.view(-1)[0] = loss_hm.float()
    loss.view(-1)[1] = loss_jt.float()
    loss.view(-1)[2] = (hm_scale * loss_hm + jt_scale * loss_jt).float()


def jointloss(x, t, w, n, kind, norm, div, loss, dx):
    with torch.enable_grad():
        xv = x.reshape(-1).detach().clone().requires_grad_(True)
        tv = t.reshape(-1)
        a, b = xv, tv
        if norm:
            a = xv / xv.abs().sum()
            b = tv / tv.abs().sum()
        d = a - b
        if kind == 0:
            l = d * d
        elif kind == 1:
            l = d.abs()
        else:
            l = torch.where(d.abs() < 1, 0.5 * d * d, d.abs() - 0.5)
        tot = (l * w.reshape(-1)).sum() / div
        tot.backward()
    if loss is not None:
        loss.view(-1)[0] = tot.detach()
    if dx is not None:
        dx.view(-1).copy_(xv.grad)


def argmax2d(hm, NJ, H, W, idx, maxval, preds):
    f = hm.reshape(NJ, H * W)
    i = f.argmax(1)
    m = f.max(1).values
    if idx is not None:
        idx.view(-1).copy_(i.int())
    if maxval is not None:
        maxval.view(-1).copy_(m)
    if preds is not None:
        mask = (m > 0).float()
        preds.view(NJ, 2).copy_(torch.stack([(i % W).float() * mask,
                                             torch.floor(i.float() / W) * mask], 1))


def adam_step(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step,
              grad_scale=1.0):
    g = grad * grad_scale
    if weight_decay:
        g = g + weight_decay * param
    exp_avg.mul_(beta1).add_(g, alpha=1 - beta1)
    exp_avg_sq.mul_(beta2).addcmul_(g, g, value=1 - beta2)
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    denom = exp_avg_sq.sqrt() / (bc2 ** 0.5) + eps
    param.addcdiv_(exp_avg, denom, value=-lr / bc1)


def sgd_step(param, grad, buf, n, lr, momentum, weight_decay, nesterov, first_step,
             grad_scale=1.0):
    g = grad * grad_scale
    if weight_decay:
        g = g + weight_decay * param
    if momentum:
        if first_step:
            buf.copy_(g)
        else:
            buf.mul_(momentum).add_(g)
        g = g + momentum * buf if nesterov else buf
    param.add_(g, alpha=-lr)


def adam_step_dev(param, grad, exp_avg, exp_avg_sq, n, hyper, step_dev):
    lr, b1, b2, eps, wd, gs = [float(v) for v in hyper]
    adam_step(param, grad, exp_avg, exp_avg_sq, n, lr, b1, b2, eps, wd, int(step_dev), gs)


def sgd_step_dev(param, grad, buf, n, hyper, step_dev):
    lr, mom, wd, nest, gs = [float(v) for v in hyper]
    sgd_step(param, grad, buf, n, lr, mom, wd, nest != 0, int(step_dev) == 1, gs)


def device_check():
    pass


def h36m_eval(pred, gt, cam, S, J, root, j14mask, pck_thr, metrics, per_joint, pck, poses):
    """CPU emulation of epb_h36m_eval: closed-form restatement in torch float64 (batched SVD)."""
    p, q, c = pred.reshape(S, J, 3).double(), gt.reshape(S, J, 3).double(), cam.reshape(S, 5).double()

    def bp(a):
        d = a[:, :, 2] + c[:, 4:5]
        return torch.stack([(a[:, :, 0] - c[:, 2:3]) / c[:, 0:1] * d,
                            (a[:, :, 1] - c[:, 3:4]) / c[:, 1:2] * d, d], dim=2)
    X, Y = bp(q), bp(p)
    muX, muY = X.mean(1, keepdim=True), Y.mean(1, keepdim=True)
    X0, Y0 = X - muX, Y - muY
    nX = X0.pow(2).sum((1, 2), keepdim=True).sqrt()
    nY = Y0.pow(2).sum((1, 2), keepdim=True).sqrt()
    A = (X0 / nX).transpose(1, 2) @ (Y0 / nY)
    U, sv, Vt = torch.linalg.svd(A)
    V = Vt.transpose(1, 2).clone()
    T = V @ U.transpose(1, 2)
    sgn = torch.sign(torch.linalg.det(T))
    V[:, :, -1] *= sgn[:, None]
    sv = sv.clone()
    sv[:, -1] *= sgn
    T = V @ U.transpose(1, 2)
    b = (sv.sum(1).reshape(S, 1, 1) * nX / nY)
    cv = muX - b * (muY @ T)
    Ya = b * (Y @ T) + cv
    Yn = b * Y
    r = lambda a: a - a[:, root:root + 1, :]
    G, P0, Pa, Pn = r(X), r(Y), r(Ya), r(Yn)
    e, ea, en = (G - P0).norm(dim=2), (G - Pa).norm(dim=2), (G - Pn).norm(dim=2)
    sel = [j for j in range(J) if (j14mask >> j) & 1]
    out = torch.stack([e.mean(1), ea.mean(1), en.mean(1), e[:, sel].mean(1), ea[:, sel].mean(1),
                       en[:, sel].mean(1), (G - P0)[:, :, 0].abs().mean(1),
                       (G - P0)[:, :, 1].abs().mean(1), (G - P0)[:, :, 2].abs().mean(1)], dim=1)
    metrics.view(S, 9).copy_(out)
    if per_joint is not None:
        per_joint.view(S, J).copy_(e)
    if pck is not None:
        pck.view(S, J).copy_((e < pck_thr).to(torch.int32))
    if poses is not None:
        poses.view(S, J, 9).copy_(torch.cat([P0, Pa, G], dim=2))


def patch_sample(img_base, img_off, img_hwp, box, flip, color, mean_std, B, patch_w, patch_h, out, trans):
    """CPU emulation of epb_patch_sample through the numpy oracle (test infrastructure)."""
    from oracle import restate
    base = img_base.numpy().reshape(-1)
    for b in range(B):
        H, W, pitch = [int(v) for v in img_hwp[b]]
        off = int(img_off[b])
        img = np.lib.stride_tricks.as_strided(base[off:], shape=(H, W, 3), strides=(pitch, 3, 1))
        bx = box[b].numpy()
        fl = bool(flip[b]) if flip is not None else False
        cs = color[b].numpy() if color is not None else np.ones(3, np.float32)
        mean = None if mean_std is None else np.asarray(mean_std[:3], dtype=np.float64)
        std = None if mean_std is None else np.asarray(mean_std[3:], dtype=np.float64)
        t, _, _, tr = restate.patch_sample(img, bx[0], bx[1], bx[2], bx[3], np.zeros((1, 3)), np.zeros((1, 3)),
                                           patch_w, patch_h, 2000.0, mean, std, bx[4], bx[5], fl, cs)
        out[b].copy_(torch.from_numpy(t))
        if trans is not None:
            trans[b].copy_(torch.from_numpy(tr.reshape(-1)))


def patch_sample_occ(img_base, img_off, img_hwp, box, flip, color, mean_std, B, patch_w, patch_h,
                     occ_base, occ_desc, occ_count, out, trans):
    """CPU emulation of epb_patch_sample_occ through the numpy oracle (test infrastructure)."""
    from oracle import restate
    base = img_base.numpy().reshape(-1)
    ob = occ_base.numpy().reshape(-1) if occ_base is not None else None
    for b in range(B):
        H, W, pitch = [int(v) for v in img_hwp[b]]
        off = int(img_off[b])
        img = np.lib.stride_tricks.as_strided(base[off:], shape=(H, W, 3), strides=(pitch, 3, 1))
        bx = box[b].numpy()
        fl = bool(flip[b]) if flip is not None else False
        cs = color[b].numpy() if color is not None else np.ones(3, np.float32)
        mean = None if mean_std is None else np.asarray(mean_std[:3], dtype=np.float64)
        std = None if mean_std is None else np.asarray(mean_std[3:], dtype=np.float64)
        occ = []
        if ob is not None:
            for k in range(int(occ_count[b])):
                o, w, h, cx, cy = [int(v) for v in occ_desc[b, k]]
                occ.append((ob[o:o + w * h * 4].reshape(h, w, 4), (cx, cy)))
        t, _, _, tr = restate.patch_sample(img, bx[0], bx[1], bx[2], bx[3], np.zeros((1, 3)), np.zeros((1, 3)),
                                           patch_w, patch_h, 2000.0, mean, std, bx[4], bx[5], fl, cs,
                                           occluders=occ)
        out[b].copy_(torch.from_numpy(t))
        if trans is not None:
            trans[b].copy_(torch.from_numpy(tr.reshape(-1)))


def patch_joints(joints, box, trans, B, J, patch_w, patch_h, rect_3d_w, depth_in_image, label):
    jt = joints.reshape(B, J, 3).double()
    M = trans.reshape(B, 2, 3).double()
    xy = torch.einsum("brc,bjc->bjr", M, torch.cat([jt[:, :, :2], torch.ones(B, J, 1, dtype=torch.float64)], 2))
    den = (box[:, 2] * box[:, 4]) if depth_in_image else (rect_3d_w * box[:, 4])
    z = jt[:, :, 2] / den.reshape(B, 1) * patch_w
    lab = torch.stack([xy[:, :, 0] / patch_w - 0.5, xy[:, :, 1] / patch_h - 0.5, z / patch_w], dim=2)
    label.view(B, J * 3).copy_(lab.reshape(B, J * 3))


def add3(a, b, c, out, n):
    r = a.reshape(-1)[:n] + b.reshape(-1)[:n]
    if c is not None:
        r = r + c.reshape(-1)[:n]
    out.view(-1)[:n].copy_(r)


def mask_scale(x, mask, scale, out, n):
    out.view(-1)[:n].copy_(torch.where(mask.reshape(-1)[:n] != 0, x.reshape(-1)[:n] * scale,
                                       torch.zeros(n, dtype=x.dtype)))


# ------------------------------------------------------------------ split-fp16 ("f16x3") family
# CPU emulation written from the contracts in include/epb.h: a split tensor is a float16
# tensor [2, ...] (hi, lo) plus sc = (s, 1/s); products are formed from the exact fp16 planes
# with the three-term rule (lo*hi + hi*lo + hi*hi) accumulated in float64.

def _split(v, s):
    v = (v.float() * s).clamp(-65504.0, 65504.0)
    hi = v.half()
    lo = (v - hi.float()).half()
    return hi, lo


def _join(t, sc):
    return (t[0].float() + t[1].float()) * float(sc[1])


def _store_split(dst, v, s):
    hi, lo = _split(v, s)
    dst[0].view(-1).copy_(hi.reshape(-1))
    dst[1].view(-1).copy_(lo.reshape(-1))


def _pow2_scale(amax):
    import math
    if not (amax > 0) or not math.isfinite(amax):
        return 1.0
    _, e = math.frexp(amax)
    k = max(-100, min(100, 13 - (e - 1)))
    return math.ldexp(1.0, k)


def act_scale(stats, scale, shift, M, C, stats2, scale2, shift2, res_sc, sc):
    import math

    # split16.cu channel_bound: kappa u is the rounding of the conv16 epilogue's fp32 sums
    ku = (16.0 + math.ceil(M / (16.0 * 132))) * 2.0 ** -24

    def grp(st, a, b):
        mean, q = st[:C] / M, st[C:] / M
        var = (q - mean * mean).clamp_min(0)
        dev = torch.sqrt(M * (var + 4.0 * ku * q)) + ku * torch.sqrt(q)
        return float(((a.double() * mean + b.double()).abs() + a.double().abs() * dev).max())
    bound = grp(stats, scale, shift)
    if stats2 is not None:
        bound += grp(stats2, scale2, shift2)
    bound = bound * 1.001 + (float(res_sc[2]) if res_sc is not None else 0.0)
    s = 1.0
    if bound > 0:
        _, e = math.frexp(bound)
        s = math.ldexp(1.0, max(-100, min(100, 15 - e)))
    sc[0], sc[1], sc[2], sc[3] = s, 1.0 / s, bound, 0.0


def bn_finalize_scale(stats, M, C, gamma, beta, eps, momentum, running_mean, running_var, scale, shift,
                      mean, invstd, stats2, scale2, shift2, res_sc, sc):
    bn_finalize(stats, M, C, gamma, beta, eps, momentum, running_mean, running_var, scale, shift, mean,
                invstd)
    act_scale(stats, scale, shift, M, C, stats2, scale2, shift2, res_sc, sc)


def bn_act_split(x, scale, shift, r, rscale, rshift, r_split, r_sc, relu, M, C, y, y_sc, mask_bits=None):
    v = x.reshape(M, C)
    if scale is not None:
        v = v * scale + shift
    if r is not None:
        q = r.reshape(M, C)
        if rscale is not None:
            q = q * rscale + rshift
        v = v + q
    elif r_split is not None:
        v = v + _join(r_split, r_sc).reshape(M, C)
    if mask_bits is not None:
        import numpy as np
        mask_bits.copy_(torch.from_numpy(np.packbits((v > 0).numpy().reshape(-1), bitorder="little")))
    if relu:
        v = torch.relu(v)
    _store_split(y, v, float(y_sc[0]))


def bn_relu_maxpool_split(x, scale, shift, y, y_sc, argidx, N, H, W, C):
    Ho, Wo = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
    tmp = torch.empty(N, Ho, Wo, C)
    bn_relu_maxpool(x, scale, shift, tmp, argidx, N, H, W, C)
    _store_split(y, tmp, float(y_sc[0]))


def im2col_split(img, col, col_sc, N, C, Hi, Wi, kh, kw, stride, pad, Ho, Wo, Kpad):
    x = img.reshape(N, C, Hi, Wi).permute(0, 2, 3, 1).contiguous()
    tmp = torch.empty(N, Ho, Wo, Kpad)
    im2col(x, tmp, N, Hi, Wi, C, C, kh, kw, stride, pad, Ho, Wo, Kpad)
    _store_split(col, tmp, float(col_sc[0]))


class SplitBatch:
    def __init__(self, jobs):
        self.jobs = list(jobs)


def split16_batch(batch):
    for (src, dst, sc) in batch.jobs:
        s = _pow2_scale(float(src.abs().max())) if src.numel() else 1.0
        sc[0], sc[1] = s, 1.0 / s
        n = src.numel()
        hi, lo = _split(src.reshape(-1), s)
        dst.view(-1)[:n].copy_(hi)
        dst.view(-1)[n:2 * n].copy_(lo)


def split16(src, dst, sc, amax_ws):
    split16_batch(SplitBatch([(src, dst, sc)]))


def _three_term(g, x, w, Kw):
    """phase-grid result [N,Hp,Wp,Cout] (float64, unscaled) of the three-term product."""
    xh, xl = x[0].reshape(g.N, g.Hi, g.Wi, g.Cin).double(), x[1].reshape(g.N, g.Hi, g.Wi, g.Cin).double()
    n = g.Cout * g.Tw * g.Cin
    wh = w.view(-1)[:n].view(g.Cout, g.Tw, g.Cin).double()
    wl = w.view(-1)[n:2 * n].view(g.Cout, g.Tw, g.Cin).double()
    acc = torch.zeros(g.N, g.Hp, g.Wp, g.Cout, dtype=torch.float64)
    for t in range(g.T):
        ah = _gather(g, xh, t, None, None)
        al = _gather(g, xl, t, None, None)
        bh, bl = wh[:, g.wt[t], :].T, wl[:, g.wt[t], :].T
        acc += al @ bh + ah @ bl + ah @ bh
    return acc


def conv16_fprop(g, x, x_sc, w, w_sc, out, bias=None, stats=None):
    assert g.Cin % 64 == 0 and g.Cout % 4 == 0
    acc = (_three_term(g, x, w, None) * (float(x_sc[1]) * float(w_sc[1]))).float()
    if bias is not None:
        acc = acc + bias
    o = out.view(g.N, g.Ho, g.Wo, g.Cout)
    sl = o[:, g.ph::g.os, g.pw::g.os][:, :g.Hp, :g.Wp]
    if g.accumulate:
        acc = acc + sl
    o[:, g.ph::g.os, g.pw::g.os][:, :g.Hp, :g.Wp] = acc
    if stats is not None:
        flat = acc.reshape(-1, g.Cout).double()
        stats[:g.Cout] += flat.sum(0)
        stats[g.Cout:] += (flat * flat).sum(0)


def conv16_wgrad(g, x, x_sc, dout, dout_sc, dw, ws):
    assert g.Cin % 64 == 0 and g.Cout % 64 == 0
    DW = dw.view(g.Cout, g.Tw, g.Cin)
    xh, xl = x[0].reshape(g.N, g.Hi, g.Wi, g.Cin).double(), x[1].reshape(g.N, g.Hi, g.Wi, g.Cin).double()

    def ph(p):
        return p.reshape(g.N, g.Ho, g.Wo, g.Cout)[:, g.ph::g.os, g.pw::g.os][:, :g.Hp, :g.Wp] \
            .reshape(-1, g.Cout).double()
    dh_, dl_ = ph(dout[0]), ph(dout[1])
    alpha = float(x_sc[1]) * float(dout_sc[1])
    for t in range(g.T):
        ah = _gather(g, xh, t, None, None).reshape(-1, g.Cin)
        al = _gather(g, xl, t, None, None).reshape(-1, g.Cin)
        DW[:, g.wt[t], :] += ((dh_.T @ al + dl_.T @ ah + dh_.T @ ah) * alpha).float()


def _mask16(dy, x, mask_hi, scale, shift, relu, M, C, mask_bits=None):
    g = dy.reshape(M, C)
    if mask_bits is not None:
        import numpy as np
        bits = np.unpackbits(mask_bits.numpy().reshape(-1), bitorder="little")[:M * C]
        return g * torch.from_numpy(bits.astype(np.float32)).reshape(M, C)
    if mask_hi is not None:
        return g * (mask_hi.reshape(M, C).float() > 0).float()
    if relu:
        return g * ((x.reshape(M, C) * scale + shift) > 0).float()
    return g


def bn_bwd_reduce_mx(dy, x, mask_hi, scale, shift, mean, invstd, relu, M, C, sums, maxes):
    g = _mask16(dy, x, mask_hi, scale, shift, relu, M, C)
    xh = (x.reshape(M, C) - mean) * invstd
    sums[:C] += g.double().sum(0)
    sums[C:] += (g.double() * xh.double()).sum(0)
    maxes[:C] = torch.maximum(maxes[:C], g.abs().max(0).values)
    maxes[C:] = torch.maximum(maxes[C:], xh.abs().max(0).values)


def bn_bwd_apply_split(dy, x, mask_hi, scale, shift, mean, invstd, gamma, relu, sums, maxes, M, C,
                       dz, dz_sc, dy_masked, dgamma, dbeta):
    g = _mask16(dy, x, mask_hi, scale, shift, relu, M, C)
    xh = (x.reshape(M, C) - mean) * invstd
    k0 = gamma * invstd
    k1 = (sums[:C] / M).float()
    k2 = (sums[C:] / M).float()
    bound = float((k0.abs() * (maxes[:C] + k1.abs() + maxes[C:] * k2.abs())).max())
    s = _pow2_scale(bound)
    dz_sc[0], dz_sc[1] = s, 1.0 / s
    maxes[:C] = k1
    maxes[C:] = k2
    v = k0 * (g - k1 - xh * k2)
    assert float(v.abs().max()) <= bound * (1 + 1e-5) + 1e-30, "dz exceeds its bound"
    _store_split(dz, v, s)
    if dy_masked is not None:
        dy_masked.view(M, C).copy_(g)
    if dgamma is not None:
        dgamma.copy_(sums[C:].float())
    if dbeta is not None:
        dbeta.copy_(sums[:C].float())


def bn_bwd_split(dy, x, mask_hi, scale, shift, mean, invstd, gamma, relu, M, C, dz, dz_sc, dy_masked,
                 dgamma, dbeta, mask_bits=None):
    sums = torch.zeros(2 * C, dtype=torch.float64)
    maxes = torch.zeros(2 * C)
    if mask_bits is not None:
        # same arithmetic on the gradient masked by the bits (dy_masked may alias dy)
        g = _mask16(dy, x, None, scale, shift, 0, M, C, mask_bits).reshape(dy.shape).clone()
        bn_bwd_reduce_mx(g, x, None, scale, shift, mean, invstd, 0, M, C, sums, maxes)
        bn_bwd_apply_split(g, x, None, scale, shift, mean, invstd, gamma, 0, sums, maxes, M, C,
                           dz, dz_sc, None, dgamma, dbeta)
        if dy_masked is not None:
            dy_masked.view(M, C).copy_(g.view(M, C))
        return
    bn_bwd_reduce_mx(dy, x, mask_hi, scale, shift, mean, invstd, relu, M, C, sums, maxes)
    bn_bwd_apply_split(dy, x, mask_hi, scale, shift, mean, invstd, gamma, relu, sums, maxes, M, C,
                       dz, dz_sc, dy_masked, dgamma, dbeta)


def avgpool_split(x, x_sc, y, N, HW, C):
    y.view(N, C).copy_(_join(x, x_sc).reshape(N, HW, C).mean(1))


def final_preds(hm, N, J, H, W, center, scale, post_process, preds, maxvals):
    from oracle import restate
    p, m = restate.final_preds(hm.reshape(N, J, H, W).numpy(), center.numpy(), scale.numpy(),
                               bool(post_process))
    preds.view(N, J, 2).copy_(torch.from_numpy(p))
    if maxvals is not None:
        maxvals.view(N, J).copy_(torch.from_numpy(m.reshape(N, J)))


def sumsq(x, n, total):
    total += (x.reshape(-1)[:n].double() ** 2).sum()


def clip_scale(x, n, total, max_norm):
    coef = max_norm / (float(total.reshape(-1)[0]) ** 0.5 + 1e-6)
    if coef < 1.0:
        x.view(-1)[:n].mul_(float(np.float32(coef)))


def patch_to_image(coords, box, B, J, patch_w, patch_h, rect3d_w, kps):
    """CPU emulation of epb_patch_to_image through the numpy oracle: soft-argmax coordinates ->
    image-frame keypoints (integral_loss.py:196-205 + img_utils.py:141-155)."""
    from oracle import restate
    res = restate.joint_location_result(patch_w, patch_h, coords.reshape(B, J * 3).numpy())
    bx = box.reshape(B, 6).numpy()
    out = np.stack([restate.trans_coords_from_patch_to_org_3d(
        res[i], bx[i, 0], bx[i, 1], bx[i, 2], bx[i, 3], patch_w, patch_h, rect3d_w, rect3d_w,
        scale=bx[i, 4], rot=bx[i, 5]) for i in range(B)])
    kps.view(B, J, 4).copy_(torch.from_numpy(out))
