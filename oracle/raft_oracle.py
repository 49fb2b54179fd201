"""CPU oracle for the RAFT-NCUP per-iteration hot path.  TEST INFRASTRUCTURE ONLY.

This file restates, as plain functional fp32 torch-CPU code, the algorithm of the
reference (abdo-eldesokey/RAFT-NCUP @ 51ac387).  It is the *checker*: only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import it.  The product path
(``raft-ncup_b200/``) never imports anything from ``oracle/``.

Parity pinning: the reference ships no tests / golden vectors (SURVEY.md §4), so
the oracle is pinned against outputs of the reference itself, generated in the
authoring container by ``oracle/make_golden.py`` (imports /root/reference) and
committed under ``tests/golden/``; ``tests/test_oracle_golden.py`` replays them.

Every function cites the reference file:line it follows.  All weights are read
from a dict that uses the reference's ``state_dict`` key names.
"""
import math

import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------- helpers


def coords_grid(batch, ht, wd):
    """core/utils/utils.py:76-79 — channel 0 = x index, channel 1 = y index."""
    ys, xs = torch.meshgrid(torch.arange(ht), torch.arange(wd), indexing="ij")
    return torch.stack([xs, ys], dim=0).float()[None].repeat(batch, 1, 1, 1)


def input_pad(dims, mode="sintel"):
    """core/utils/utils.py:7-19 — (left, right, top, bottom) replicate padding to a multiple of 8."""
    ht, wd = dims[-2:]
    pad_ht = (((ht // 8) + 1) * 8 - ht) % 8
    pad_wd = (((wd // 8) + 1) * 8 - wd) % 8
    if mode == "sintel":
        return [pad_wd // 2, pad_wd - pad_wd // 2, pad_ht // 2, pad_ht - pad_ht // 2]
    return [pad_wd // 2, pad_wd - pad_wd // 2, 0, pad_ht]


def pad_images(pad, *imgs):
    """core/utils/utils.py:21-22."""
    return [F.pad(x, pad, mode="replicate") for x in imgs]


def unpad(pad, x):
    """core/utils/utils.py:24-27."""
    ht, wd = x.shape[-2:]
    return x[..., pad[2]:ht - pad[3], pad[0]:wd - pad[1]]


# --------------------------------------------------------------------------- A1/A2/A3: correlation


def corr_pyramid(fmap1, fmap2, num_levels=4):
    """core/corr.py:7-21,47-55 — all-pairs volume / sqrt(D), then (levels-1) 2x2 average pools."""
    b, d, h, w = fmap1.shape
    vol = torch.matmul(fmap1.reshape(b, d, h * w).transpose(1, 2), fmap2.reshape(b, d, h * w))
    vol = vol / math.sqrt(float(d))
    vol = vol.reshape(b * h * w, 1, h, w)
    pyr = [vol]
    for _ in range(num_levels - 1):
        vol = F.avg_pool2d(vol, 2, stride=2)
        pyr.append(vol)
    return pyr


def _bilinear_zero(img, x, y, round_trip=True):
    """core/utils/utils.py:59-73 (grid_sample, bilinear, align_corners=True, zeros padding) written
    out by hand.  img [N,1,H,W]; x,y [N,K] pixel coordinates.  Includes the reference's
    pixel -> [-1,1] -> pixel round trip so that fp32 rounding of the sample position matches
    (round_trip=False: sample at x, y themselves, as the kernels do)."""
    n, _, h, w = img.shape
    if round_trip:
        xn = 2 * x / (w - 1) - 1
        yn = 2 * y / (h - 1) - 1
        x = ((xn + 1) / 2) * (w - 1)
        y = ((yn + 1) / 2) * (h - 1)
    x0 = torch.floor(x)
    y0 = torch.floor(y)
    ax = x - x0
    ay = y - y0
    flat = img.reshape(n, h * w)
    out = torch.zeros_like(x)
    for dy, wy in ((0, 1 - ay), (1, ay)):
        for dx, wx in ((0, 1 - ax), (1, ax)):
            xi = x0 + dx
            yi = y0 + dy
            ok = (xi >= 0) & (xi <= w - 1) & (yi >= 0) & (yi <= h - 1)
            idx = (yi.clamp(0, h - 1) * w + xi.clamp(0, w - 1)).long()
            out = out + torch.gather(flat, 1, idx) * (wx * wy) * ok.float()
    return out


def corr_lookup(pyr, coords, radius=4, dtype=torch.float32, round_trip=True):
    """core/corr.py:23-44 — channel k = l*(2r+1)^2 + i*(2r+1) + j samples level l at
    x = cx/2^l + (i-r), y = cy/2^l + (j-r): the SLOW window index offsets x (corr.py:31-37).
    dtype: of the result (torch.float64 keeps an fp64 evaluation in fp64).  round_trip: see _bilinear_zero; an fp64
    reference of the kernels leaves it out, or a window edge on an exact integer position gets a weight of ~1e-14
    outside the image where the kernels (and exact arithmetic) give 0."""
    b, _, h, w = coords.shape
    n = b * h * w
    side = 2 * radius + 1
    c = coords.permute(0, 2, 3, 1).reshape(n, 2)
    d = torch.arange(-radius, radius + 1, dtype=torch.float32, device=coords.device)
    off_i = d.view(side, 1).expand(side, side).reshape(1, -1)  # added to x
    off_j = d.view(1, side).expand(side, side).reshape(1, -1)  # added to y
    outs = []
    for lvl, vol in enumerate(pyr):
        cx = c[:, 0:1] / 2 ** lvl + off_i
        cy = c[:, 1:2] / 2 ** lvl + off_j
        outs.append(_bilinear_zero(vol, cx, cy, round_trip).view(b, h, w, side * side))
    return torch.cat(outs, dim=-1).permute(0, 3, 1, 2).contiguous().to(dtype)


def corr_lookup_direct(fmap1, fmap2, coords, num_levels=4, radius=4):
    """SURVEY.md Appendix A.1 — same result as corr_pyramid+corr_lookup without the 4-D volume:
    pooling commutes with the dot product, so level l correlates fmap1 against avg-pooled fmap2."""
    b, d, h, w = fmap1.shape
    side = 2 * radius + 1
    f1 = fmap1.permute(0, 2, 3, 1).reshape(b, h * w, d)
    dev = fmap1.device               # (device- and dtype-agnostic: the GPU tests evaluate it in fp64 on the device)
    out = torch.zeros(b, h * w, num_levels * side * side, dtype=fmap1.dtype, device=dev)
    f2 = fmap2
    for lvl in range(num_levels):
        hl, wl = f2.shape[-2:]
        f2l = f2.permute(0, 2, 3, 1)  # [b,hl,wl,d]
        cx = coords[:, 0].reshape(b, h * w) / 2 ** lvl
        cy = coords[:, 1].reshape(b, h * w) / 2 ** lvl
        x0 = torch.floor(cx)
        y0 = torch.floor(cy)
        ax = (cx - x0)[..., None, None]
        ay = (cy - y0)[..., None, None]
        g = torch.zeros(b, h * w, side + 1, side + 1, dtype=fmap1.dtype, device=dev)  # G[a][c]: a -> x lattice, c -> y lattice
        for a in range(side + 1):
            for c in range(side + 1):
                xi = x0 - radius + a
                yi = y0 - radius + c
                ok = (xi >= 0) & (xi <= wl - 1) & (yi >= 0) & (yi <= hl - 1)
                xi = xi.clamp(0, wl - 1).long()
                yi = yi.clamp(0, hl - 1).long()
                bi = torch.arange(b, device=dev)[:, None].expand(b, h * w)
                v = f2l[bi, yi, xi]  # [b,P,d]
                g[:, :, a, c] = (v * f1).sum(-1) * ok.float() / math.sqrt(float(d))
        blend = ((1 - ax) * (1 - ay) * g[:, :, :-1, :-1] + ax * (1 - ay) * g[:, :, 1:, :-1]
                 + (1 - ax) * ay * g[:, :, :-1, 1:] + ax * ay * g[:, :, 1:, 1:])
        out[:, :, lvl * side * side:(lvl + 1) * side * side] = blend.reshape(b, h * w, side * side)
        if lvl + 1 < num_levels:
            f2 = F.avg_pool2d(f2, 2, stride=2)
    return out.view(b, h, w, -1).permute(0, 3, 1, 2).contiguous()


# --------------------------------------------------------------------------- A5..A8: update block


def _conv(sd, name, x, padding):
    return F.conv2d(x, sd[name + ".weight"], sd[name + ".bias"], padding=padding)


def motion_encoder(sd, flow, corr, p="update_block.encoder."):
    """core/update.py:79-97."""
    cor = F.relu(_conv(sd, p + "convc1", corr, 0))
    cor = F.relu(_conv(sd, p + "convc2", cor, 1))
    flo = F.relu(_conv(sd, p + "convf1", flow, 3))
    flo = F.relu(_conv(sd, p + "convf2", flo, 1))
    out = F.relu(_conv(sd, p + "conv", torch.cat([cor, flo], 1), 1))
    return torch.cat([out, flow], 1)


def sep_conv_gru(sd, h, x, p="update_block.gru."):
    """core/update.py:33-60 — (1x5) half step then (5x1) half step."""
    for tag, pad in (("1", (0, 2)), ("2", (2, 0))):
        hx = torch.cat([h, x], 1)
        z = torch.sigmoid(_conv(sd, p + "convz" + tag, hx, pad))
        r = torch.sigmoid(_conv(sd, p + "convr" + tag, hx, pad))
        q = torch.tanh(_conv(sd, p + "convq" + tag, torch.cat([r * h, x], 1), pad))
        h = (1 - z) * h + z * q
    return h


def flow_head(sd, net, p="update_block.flow_head."):
    """core/update.py:6-14."""
    return _conv(sd, p + "conv2", F.relu(_conv(sd, p + "conv1", net, 1)), 1)


def mask_head(sd, net, p="update_block.mask."):
    """core/update.py:123-126,140 (model `raft` only): 0.25 * conv1x1(relu(conv3x3(net)))."""
    return 0.25 * _conv(sd, p + "2", F.relu(_conv(sd, p + "0", net, 1)), 0)


def update_block(sd, net, inp, corr, flow, with_mask):
    """core/update.py:130-141.  Returns (net, mask|None, delta_flow)."""
    motion = motion_encoder(sd, flow, corr)
    net = sep_conv_gru(sd, net, torch.cat([inp, motion], 1))
    delta = flow_head(sd, net)
    mask = mask_head(sd, net) if with_mask else None
    return net, mask, delta


# --------------------------------------------------------------------------- U1: convex upsampler


def convex_upsample(flow, mask):
    """core/raft.py:73-84 — softmax over the 9 neighbours, weighted sum of unfold(8*flow)."""
    n, _, h, w = flow.shape
    m = torch.softmax(mask.view(n, 1, 9, 8, 8, h, w), dim=2)
    nb = F.unfold(8 * flow, [3, 3], padding=1).view(n, 2, 9, 1, 1, h, w)
    up = torch.sum(m * nb, dim=2).permute(0, 1, 4, 2, 5, 3)
    return up.reshape(n, 2, 8 * h, 8 * w)


# --------------------------------------------------------------------------- U2..U6: NCUP


def softplus10(p):
    """core/nconv_modules.py:263-264 — W = softplus(weight_p, beta=10), recomputed every forward."""
    return F.softplus(p, beta=10)


def nconv2d(data, conf, weight, eps=1e-20):
    """core/nconv_modules.py:164-199 — normalized convolution + confidence propagation (no bias)."""
    pad = weight.shape[-1] // 2
    den = F.conv2d(conf, weight, None, 1, pad)
    num = F.conv2d(data * conf, weight, None, 1, pad)
    y = num / (den + eps)
    s = weight.reshape(weight.shape[0], -1).sum(-1).view(1, -1, 1, 1)
    return y, den / s


def zero_stuff(x, scale=4):
    """core/upsampler.py:179-210 — zeros [B,C,s*h,s*w] with out[..., s//2::s, s//2::s] = x."""
    b, c, h, w = x.shape
    out = torch.zeros(b, c, h * scale, w * scale, dtype=x.dtype, device=x.device)
    out[:, :, scale // 2::scale, scale // 2::scale] = x
    return out


def weights_net(sd, x, use_bn, p="upsampler.weights_est_net."):
    """core/interp_weights_est.py:10-47 (Simple, num_ch [130,64,32], filters [3,3,1]) followed by the
    sigmoid final_act wired in core/upsampler.py:44-46.  BatchNorm in eval mode (running stats)."""
    for i in range(2):
        x = F.conv2d(x, sd[f"{p}conv.{i}.0.weight"], sd[f"{p}conv.{i}.0.bias"], padding=1)
        if use_bn:
            x = F.batch_norm(x, sd[f"{p}conv.{i}.1.running_mean"], sd[f"{p}conv.{i}.1.running_var"],
                             sd[f"{p}conv.{i}.1.weight"], sd[f"{p}conv.{i}.1.bias"], False, 0.0, 1e-5)
        x = F.relu(x)
    return torch.sigmoid(F.conv2d(x, sd[p + "out.weight"], sd[p + "out.bias"]))


def nconv_unet_live(sd, data, conf, p="upsampler.interpolation_net."):
    """core/nconv_modules.py:106-136 at the shipped config (num_downsampling=1): the decoder consumes
    x[1] twice (index quirk at :128-131) so the pooled branch is dead; live path = nconv_in ->
    nconv_x2[0] -> decoder[0](cat(x1,x1)) -> nconv_out (SURVEY.md Appendix A.3)."""
    w1 = softplus10(sd[p + "nconv_in.weight_p"])
    w2 = softplus10(sd[p + "nconv_x2.0.weight_p"])
    w3 = softplus10(sd[p + "decoder.0.weight_p"])
    w4 = softplus10(sd[p + "nconv_out.weight_p"])
    x, c = nconv2d(data, conf, w1)
    x, c = nconv2d(x, c, w2)
    x, c = nconv2d(torch.cat([x, x], 1), torch.cat([c, c], 1), w3)
    x, c = nconv2d(x, c, w4)
    return x, c


def ncup_upsample(sd, flow_lr, guidance, use_bn=True, return_conf=False):
    """core/raft_nc_dbl.py:107-112 + core/upsampler.py:143-177: nearest x2, weights net on
    cat(flow x2, guidance x2), zero-stuffed data/confidence (scale 4, offset 2), channels->batch NConv."""
    x4 = F.interpolate(flow_lr, scale_factor=2, mode="nearest")
    g4 = F.interpolate(guidance, x4.shape[2:], mode="area")
    w4 = weights_net(sd, torch.cat([x4, g4], 1), use_bn)
    xh = zero_stuff(x4)
    wh = zero_stuff(w4)
    b, c, oh, ow = xh.shape
    out, _ = nconv_unet_live(sd, xh.view(b * c, 1, oh, ow), wh.view(b * c, 1, oh, ow))
    out = out.view(b, c, oh, ow)
    return (out, w4) if return_conf else out


# --------------------------------------------------------------------------- C6: encoders


def _norm(sd, name, x, kind):
    if kind == "instance":
        return F.instance_norm(x)  # nn.InstanceNorm2d default: affine=False, no running stats
    if kind == "batch":
        return F.batch_norm(x, sd[name + ".running_mean"], sd[name + ".running_var"],
                            sd[name + ".weight"], sd[name + ".bias"], False, 0.0, 1e-5)
    raise ValueError(kind)


def _res_block(sd, p, x, kind, stride):
    """core/extractor.py:6-56."""
    y = F.relu(_norm(sd, p + "norm1", F.conv2d(x, sd[p + "conv1.weight"], sd[p + "conv1.bias"], stride, 1), kind))
    y = F.relu(_norm(sd, p + "norm2", F.conv2d(y, sd[p + "conv2.weight"], sd[p + "conv2.bias"], 1, 1), kind))
    if stride != 1:
        x = F.conv2d(x, sd[p + "downsample.0.weight"], sd[p + "downsample.0.bias"], stride)
        x = _norm(sd, p + "downsample.1", x, kind)
    return F.relu(x + y)


def basic_encoder(sd, p, x, kind):
    """core/extractor.py:118-192 (eval mode, dropout 0)."""
    x = F.conv2d(x, sd[p + "conv1.weight"], sd[p + "conv1.bias"], 2, 3)
    x = F.relu(_norm(sd, p + "norm1", x, kind))
    for layer, stride in (("layer1", 1), ("layer2", 2), ("layer3", 2)):
        x = _res_block(sd, f"{p}{layer}.0.", x, kind, stride)
        x = _res_block(sd, f"{p}{layer}.1.", x, kind, 1)
    return F.conv2d(x, sd[p + "conv2.weight"], sd[p + "conv2.bias"])


# --------------------------------------------------------------------------- A9: the model loop


def raft_forward_graph(sd, image1, image2, iters=12, model="raft_nc_dbl", flow_init=None, use_bn=True,
                       upsample_every_iter=True, trace=None):
    """core/raft_nc_dbl.py:115-173 (model='raft_nc_dbl') / core/raft.py:87-143 (model='raft').
    Returns (flow_low, flow_up_last, [flow_up per iter]).  `trace`, if a dict, receives teacher-forcing
    tensors.  upsample_every_iter=False skips the (result-irrelevant) per-iteration NCUP calls the
    reference makes in test_mode (raft_nc_dbl.py:161).
    Differentiable when the tensors of `sd` require grad (training oracle, train.py:215: BatchNorm in eval mode as after
    freeze_bn(), train.py:185-186); `coords1` is detached at the top of every iteration like raft_nc_dbl.py:149."""
    image1 = (2 * (image1 / 255.0) - 1.0).contiguous()
    image2 = (2 * (image2 / 255.0) - 1.0).contiguous()
    b = image1.shape[0]
    fmaps = basic_encoder(sd, "fnet.", torch.cat([image1, image2], 0), "instance").float()
    fmap1, fmap2 = fmaps[:b], fmaps[b:]
    pyr = corr_pyramid(fmap1, fmap2)
    cnet = basic_encoder(sd, "cnet.", image1, "batch")
    net, inp = torch.tanh(cnet[:, :128]), torch.relu(cnet[:, 128:])
    h8, w8 = image1.shape[2] // 8, image1.shape[3] // 8
    coords0 = coords_grid(b, h8, w8).to(image1.device)     # (device-agnostic: the tests also evaluate this graph in fp32 on the GPU)
    coords1 = coords_grid(b, h8, w8).to(image1.device)
    if flow_init is not None:
        coords1 = coords1 + flow_init
    if trace is not None:
        trace.update(fmap1=fmap1, fmap2=fmap2, net0=net, inp=inp, iters=[])
    ups = []
    flow_up = None
    for it in range(iters):
        coords1 = coords1.detach()
        corr = corr_lookup(pyr, coords1)
        flow = coords1 - coords0
        net, mask, delta = update_block(sd, net, inp, corr, flow, with_mask=(model == "raft"))
        coords_in = coords1
        coords1 = coords1 + delta
        last = it == iters - 1
        if model == "raft":
            flow_up = convex_upsample(coords1 - coords0, mask)
        elif upsample_every_iter or last:
            flow_up = 8 * ncup_upsample(sd, coords1 - coords0, net, use_bn)
        ups.append(flow_up)
        if trace is not None:
            trace["iters"].append(dict(coords=coords_in, corr=corr, net=net, delta=delta, mask=mask, flow_up=flow_up))
    return coords1 - coords0, flow_up, ups


raft_forward = torch.no_grad()(raft_forward_graph)


def forward_interpolate(flow):
    """core/utils/utils.py:28-56 — push pixels along the flow, keep samples strictly inside the image, nearest-sample
    interpolation back onto the grid (scipy griddata 'nearest', fill 0).  flow: [2,H,W] tensor; returns a [2,H,W] tensor."""
    import numpy as np
    from scipy import interpolate
    f = flow.detach().cpu().numpy()
    dx, dy = f[0], f[1]
    ht, wd = dx.shape
    x0, y0 = np.meshgrid(np.arange(wd), np.arange(ht))
    x1, y1 = (x0 + dx).reshape(-1), (y0 + dy).reshape(-1)
    dxr, dyr = dx.reshape(-1), dy.reshape(-1)
    ok = (x1 > 0) & (x1 < wd) & (y1 > 0) & (y1 < ht)
    fx = interpolate.griddata((x1[ok], y1[ok]), dxr[ok], (x0, y0), method="nearest", fill_value=0)
    fy = interpolate.griddata((x1[ok], y1[ok]), dyr[ok], (x0, y0), method="nearest", fill_value=0)
    return torch.from_numpy(np.stack([fx, fy], 0)).float()


def sequence_loss(flow_preds, flow_gt, valid, gamma=0.8, max_flow=400.0):
    """train.py:46-71 — gamma-weighted L1 over all predictions; invalid pixels count in the mean's denominator."""
    n = len(flow_preds)
    mag = torch.sum(flow_gt ** 2, dim=1).sqrt()
    valid = (valid >= 0.5) & (mag < max_flow)
    loss = 0.0
    for i, pred in enumerate(flow_preds):
        loss = loss + gamma ** (n - i - 1) * (valid[:, None] * (pred - flow_gt).abs()).mean()
    return loss
