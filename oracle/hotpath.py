"""ORACLE - TEST INFRASTRUCTURE ONLY.  CPU restatement of the MVSFormer++ depth-inference hot path.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference``
legs may import this package.  The product path (``mvsformerplusplus_b200``) never does; it fails
loudly when the CUDA library is missing.

Every function restates one reference function in plain torch CPU ops (dtype follows the inputs, so the
same code gives an fp32 answer - the parity oracle - and an fp64 answer - the "truth" used to size
tolerances).  It is self-contained: it does NOT import /root/reference.  It is *pinned* against the
reference's own modules executed in the build container by ``oracle/gen_golden.py`` (committed
fixtures under tests/golden/, checked by tests/test_oracle_golden.py), because the reference ships no
tests or golden vectors of its own (SURVEY.md §4, §8c).

Weights are passed as a flat state dict ``sd`` with the reference's key names
(tests/golden/hotpath_state_dict_keys.txt).

Reference files restated (relative to the reference repo root):
  models/warping.py:69-109            homo_warp
  models/cost_volume.py:51-133        stage_forward (group correlation, entropy visibility, aggregation,
                                      soft-argmax, confidence)
  models/module.py:367-408,453-504    costreg_unet  (CostRegNet / CostRegNet3D)
  models/module.py:507-646            costreg_transformer (PureTransformerCostReg)
  models/dino/layers/attention.py:51-99,141-170   softmax attention with entropy-invariance scale
  models/module.py:649-655,692-724    depth_regression, init_inverse_range, schedule_inverse_range
  models/position_encoding.py:42-89,138-189  pe2d_sine_norm, get_position_3d, position_encoding_3d
  models/FMT.py:81-206, models/dino/layers/block.py:336-346, attention.py:261-291, mlp.py, layer_scale.py
                                      fmt_with_pathway
  models/networks/DINOv2_mvsformer_model.py:117-179   hotpath_forward (cascade glue)
"""
import math

import torch
import torch.nn.functional as F

# When True the two heavy gathers/contractions call the same ATen kernels the reference calls on CPU
# (F.grid_sample at warping.py:105, F.scaled_dot_product_attention at attention.py:96) instead of the explicit
# restatements below.  Used by bench.py's CPU-baseline arm so the timing reflects the reference's own CPU path;
# parity tests use the explicit restatements (and check both agree).
USE_ATEN_KERNELS = False

# The reference forms  proj = src_proj @ inverse(ref_proj)  with fp32 LAPACK (warping.py:80).  At full resolution source
# coordinates reach ~1.5e3 px, where one fp32 ulp is 1.2e-4 px: ANY re-rounding of that 4x4 product (another LAPACK, a
# GPU solver, fp64) moves white-noise feature samples by up to ~2e-3, i.e. the reference is only defined up to that noise.
# The CUDA library composes the homography in fp64 and rounds once (DESIGN.md "Numerics").  With this flag the oracle does
# the same, everything else unchanged - used by tests/test_gpu_fullsize.py to separate "kernel arithmetic" (held to the
# north-star tolerances against this variant) from "sensitivity of the reference to its own 4x4 inverse" (measured
# oracle-vs-oracle and reported as the noise floor).
HOMOGRAPHY_FP64 = False


# --------------------------------------------------------------------------------------------------
# W1/W2: projection prep + homography warp
# --------------------------------------------------------------------------------------------------
def compose_projection(proj):
    """cost_volume.py:68-71: P_new = E ; P_new[:3,:4] = K[:3,:3] @ E[:3,:4].  proj [B,2,4,4]."""
    if HOMOGRAPHY_FP64:
        proj = proj.double()   # kept in fp64 until the homography has been formed (warp_coordinates rounds once)
    new = proj[:, 0].clone()
    new[:, :3, :4] = torch.matmul(proj[:, 1, :3, :3], proj[:, 0, :3, :4])
    return new


def warp_coordinates(src_proj, ref_proj, depth_values, H, W):
    """warping.py:79-96.  Returns pixel coordinates (px, py) [B,D,H*W] as the bilinear sampler sees them
    (i.e. after the normalise -> un-normalise round trip of warping.py:94-95 + grid_sample
    align_corners=True) and z [B,D,H*W]."""
    B, D = depth_values.shape[0], depth_values.shape[1]
    dt = depth_values.dtype
    if HOMOGRAPHY_FP64:
        proj = torch.matmul(src_proj.double(), torch.inverse(ref_proj.double())).to(dt)
    else:
        proj = torch.matmul(src_proj, torch.inverse(ref_proj))
    rot, trans = proj[:, :3, :3], proj[:, :3, 3:4]
    y, x = torch.meshgrid([torch.arange(0, H, dtype=dt), torch.arange(0, W, dtype=dt)], indexing="ij")
    xyz = torch.stack((x.reshape(-1), y.reshape(-1), torch.ones(H * W, dtype=dt)))
    rot_xyz = torch.matmul(rot, xyz.unsqueeze(0).repeat(B, 1, 1))
    rot_depth_xyz = rot_xyz.unsqueeze(2) * depth_values.reshape(B, 1, D, -1)
    proj_xyz = rot_depth_xyz + trans.view(B, 3, 1, 1)
    proj_xy = proj_xyz[:, :2] / (proj_xyz[:, 2:3] + 1e-6)
    gx = proj_xy[:, 0] / ((W - 1) / 2) - 1
    gy = proj_xy[:, 1] / ((H - 1) / 2) - 1
    # grid_sample(align_corners=True) un-normalisation: ((g + 1) / 2) * (size - 1)
    px = ((gx + 1) / 2) * (W - 1)
    py = ((gy + 1) / 2) * (H - 1)
    return px, py, proj_xyz[:, 2]


def bilinear_gather_zeros(src_fea, px, py):
    """F.grid_sample(mode='bilinear', padding_mode='zeros', align_corners=True) restated as an explicit
    4-corner gather.  src_fea [B,C,H,W]; px,py [B,N] pixel coordinates -> [B,C,N]."""
    B, C, H, W = src_fea.shape
    x0f, y0f = torch.floor(px), torch.floor(py)
    wx1, wy1 = px - x0f, py - y0f
    wx0, wy0 = 1 - wx1, 1 - wy1
    flat = src_fea.reshape(B, C, H * W)
    out = torch.zeros(B, C, px.shape[1], dtype=src_fea.dtype)
    finite = torch.isfinite(px) & torch.isfinite(py)
    x0f = torch.where(finite, x0f, torch.full_like(x0f, -10.0))
    y0f = torch.where(finite, y0f, torch.full_like(y0f, -10.0))
    for dx, dy, w in ((0, 0, wx0 * wy0), (1, 0, wx1 * wy0), (0, 1, wx0 * wy1), (1, 1, wx1 * wy1)):
        xi, yi = (x0f + dx), (y0f + dy)
        valid = (xi >= 0) & (xi <= W - 1) & (yi >= 0) & (yi <= H - 1)
        idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long()
        vals = torch.gather(flat, 2, idx.unsqueeze(1).expand(B, C, -1))
        wv = torch.where(valid, w, torch.zeros_like(w))
        out = out + vals * wv.unsqueeze(1)
    return out


def homo_warp(src_fea, src_proj, ref_proj, depth_values):
    """warping.py:69-109 -> (warped [B,C,D,H,W], mask [B,D,H,W])."""
    B, C, H, W = src_fea.shape
    D = depth_values.shape[1]
    if depth_values.dim() == 2:
        depth_values = depth_values.view(B, D, 1, 1).expand(B, D, H, W)
    px, py, z = warp_coordinates(src_proj, ref_proj, depth_values, H, W)
    gx = px / ((W - 1) / 2) - 1
    gy = py / ((H - 1) / 2) - 1
    if USE_ATEN_KERNELS:
        grid = torch.stack((gx, gy), dim=3)
        warped = F.grid_sample(src_fea, grid.view(B, D * H, W, 2), mode="bilinear", padding_mode="zeros",
                               align_corners=True).view(B, C, D, H, W)
    else:
        warped = bilinear_gather_zeros(src_fea, px.reshape(B, -1), py.reshape(B, -1)).view(B, C, D, H, W)
    mask = ((gx > 1) | (gx < -1) | (gy > 1) | (gy < -1) | (z <= 0)).view(B, D, H, W)
    return warped, mask


# --------------------------------------------------------------------------------------------------
# W3/W4: group correlation, entropy visibility weights, aggregation
# --------------------------------------------------------------------------------------------------
def _bn(x, sd, p, eps=1e-5):
    shape = [1, -1] + [1] * (x.dim() - 2)
    return (x - sd[p + "running_mean"].view(shape)) / torch.sqrt(sd[p + "running_var"].view(shape) + eps) \
        * sd[p + "weight"].view(shape) + sd[p + "bias"].view(shape)


def vis_cnn(entropy, sd, p):
    """cost_volume.py:37: ConvBnReLU(1,16) ConvBnReLU(16,16) ConvBnReLU(16,8) Conv1x1(8,1) Sigmoid."""
    x = entropy
    for i in range(3):
        x = F.relu(_bn(F.conv2d(x, sd[f"{p}vis.{i}.conv.weight"], padding=1), sd, f"{p}vis.{i}.bn."))
    x = F.conv2d(x, sd[f"{p}vis.3.weight"], sd[f"{p}vis.3.bias"])
    return torch.sigmoid(x)


def group_correlation(ref_feat, warped, G):
    """cost_volume.py:78-87."""
    B, C, D, H, W = warped.shape
    if G < C:
        return (ref_feat.view(B, G, C // G, 1, H, W) * warped.view(B, G, C // G, D, H, W)).mean(dim=2)
    if G == C:
        return ref_feat.view(B, G, 1, H, W) * warped
    raise AssertionError("G must <= C!")


def cost_volume(features, proj_matrices, depth_values, sd, p, G):
    """cost_volume.py:52-101 -> dict(volume_mean [B,G,D,H,W], entropy [B,V-1,H,W], vis_weight [B,V-1,H,W])."""
    ref_feat, src_feats = features[:, 0], torch.unbind(features[:, 1:], dim=1)
    projs = torch.unbind(proj_matrices, 1)
    assert len(src_feats) == len(projs) - 1, "Different number of images and projection matrices"
    ref_new = compose_projection(projs[0])
    volume_sum, vis_sum, ents, viss = 0.0, 0.0, [], []
    for src_feat, src_proj in zip(src_feats, projs[1:]):
        warped, _ = homo_warp(src_feat, compose_projection(src_proj), ref_new, depth_values)
        in_prod = group_correlation(ref_feat, warped, G)
        sim = in_prod.sum(dim=1)
        sim_norm = F.softmax(sim, dim=1)
        entropy = (-sim_norm * torch.log(sim_norm + 1e-7)).sum(dim=1, keepdim=True)
        w = vis_cnn(entropy, sd, p)
        volume_sum = volume_sum + in_prod * w.unsqueeze(1)
        vis_sum = vis_sum + w
        ents.append(entropy[:, 0])
        viss.append(w[:, 0])
    volume_mean = volume_sum / (vis_sum.unsqueeze(1) + 1e-6)
    return dict(volume_mean=volume_mean, entropy=torch.stack(ents, 1), vis_weight=torch.stack(viss, 1))


# --------------------------------------------------------------------------------------------------
# R2-R4: 3-D conv U-Nets
# --------------------------------------------------------------------------------------------------
def costreg_unet(x, sd, p):
    """module.py:398-408 (CostRegNet, stride 2) / :494-504 (CostRegNet3D, stride (1,2,2)); the variant is
    recognised from the key names (conv7.conv.weight vs conv7.0.weight)."""
    is3d = (p + "conv7.0.weight") in sd
    s = (1, 2, 2) if is3d else (2, 2, 2)
    op = (0, 1, 1) if is3d else (1, 1, 1)

    def cbr(x, name, stride):
        return F.relu(_bn(F.conv3d(x, sd[f"{p}{name}.conv.weight"], stride=stride, padding=1), sd, f"{p}{name}.bn."))

    def dbr(x, name):
        if is3d:
            y = F.conv_transpose3d(x, sd[f"{p}{name}.0.weight"], stride=s, padding=1, output_padding=op)
            return F.relu(_bn(y, sd, f"{p}{name}.1."))
        y = F.conv_transpose3d(x, sd[f"{p}{name}.conv.weight"], stride=s, padding=1, output_padding=op)
        return F.relu(_bn(y, sd, f"{p}{name}.bn."))

    conv0 = x
    conv2 = cbr(cbr(conv0, "conv1", s), "conv2", 1)
    conv4 = cbr(cbr(conv2, "conv3", s), "conv4", 1)
    x = cbr(cbr(conv4, "conv5", s), "conv6", 1)
    x = conv4 + dbr(x, "conv7")
    x = conv2 + dbr(x, "conv9")
    x = conv0 + dbr(x, "conv11")  # inner == Identity (in_channels == base_channels)
    if is3d:
        return F.conv3d(x, sd[p + "prob.weight"], sd[p + "prob.bias"])
    return F.conv3d(x, sd[p + "prob.weight"], padding=1)


# --------------------------------------------------------------------------------------------------
# R1: transformer regulariser
# --------------------------------------------------------------------------------------------------
def position_encoding_3d(position3d, C, rescale=4.0):
    """position_encoding.py:164-189 -> [B,3C,D,H,W]."""
    B, _, D, H, W = position3d.shape
    dt = position3d.dtype
    div = torch.exp(torch.arange(0, C, 2).float() * (-math.log(10000.0) / C)).to(position3d.device, dt)[None, :, None]
    pes = []
    for a in range(3):
        pe = torch.zeros(B, C, D * H * W, dtype=dt, device=position3d.device)
        pos = position3d[:, a].reshape(B, 1, -1)
        pe[:, 0::2] = torch.sin(pos * rescale * div)
        pe[:, 1::2] = torch.cos(pos * rescale * div)
        pes.append(pe)
    return torch.cat(pes, dim=1).reshape(B, 3 * C, D, H, W)


def layer_norm_3d(x, w, b, eps=1e-6):
    """module.py:586-599 (channel dim of a 5-D tensor, biased variance)."""
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    x = (x - u) / torch.sqrt(s + eps)
    return w[:, None, None, None] * x + b[:, None, None, None]


def softmax_attention(x, qkv_w, proj_w, proj_b, num_heads, train_avg_length):
    """attention.py:76-99 (SDPA fallback == flash path :141-170): scale = hd^-0.5 * log_{train_avg_length}(N)."""
    B, N, C = x.shape
    hd = C // num_heads
    qkv = F.linear(x, qkv_w).reshape(B, N, 3, num_heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    scale = hd ** -0.5
    if train_avg_length is not None:
        scale *= math.log(N, train_avg_length)
    if USE_ATEN_KERNELS:
        x = F.scaled_dot_product_attention(q, k, v, scale=scale).transpose(1, 2).reshape(B, N, C)
        return F.linear(x, proj_w, proj_b)
    out = torch.empty_like(q)
    blk = 4096  # blocked to bound memory; same arithmetic as softmax(q k^T * scale) v
    for h in range(num_heads):
        kh, vh = k[:, h], v[:, h]
        for s0 in range(0, N, blk):
            a = torch.softmax(torch.matmul(q[:, h, s0:s0 + blk], kh.transpose(-2, -1)) * scale, dim=-1)
            out[:, h, s0:s0 + blk] = torch.matmul(a, vh)
    x = out.transpose(1, 2).reshape(B, N, C)
    return F.linear(x, proj_w, proj_b)


def costreg_transformer(x, position3d, sd, p, cfg):
    """module.py:631-646 with FlashAttnBlock post-norm (:569-582)."""
    C = x.shape[1]
    dr = tuple(cfg["down_rate"])
    if position3d is not None:
        x = x + F.conv3d(position_encoding_3d(position3d, C), sd[p + "pe_proj.weight"])
    x = F.conv3d(x, sd[p + "down.0.weight"], sd[p + "down.0.bias"], stride=dr)
    x = layer_norm_3d(x, sd[p + "down.1.weight"], sd[p + "down.1.bias"])
    b, c, d, h, w = x.shape
    tal = cfg["train_avg_length"] if cfg.get("softmax_scale") == "entropy_invariance" else None
    t = x.permute(0, 3, 4, 2, 1).reshape(b, h * w * d, c)  # "b c d h w -> b (h w d) c"
    for i in range(cfg["layer_num"]):
        q = f"{p}attention_layers.{i}."
        a = softmax_attention(t, sd[q + "attn.qkv.weight"], sd[q + "attn.proj.weight"], sd[q + "attn.proj.bias"],
                              cfg["num_heads"], tal)
        t = F.layer_norm(t + sd[q + "gamma1"] * a, (c,), sd[q + "norm1.weight"], sd[q + "norm1.bias"], 1e-5)
        f = F.linear(F.gelu(F.linear(t, sd[q + "ffn.linear1.weight"], sd[q + "ffn.linear1.bias"])),
                     sd[q + "ffn.linear2.weight"], sd[q + "ffn.linear2.bias"])
        t = F.layer_norm(t + sd[q + "gamma2"] * f, (c,), sd[q + "norm2.weight"], sd[q + "norm2.bias"], 1e-5)
    x = t.reshape(b, h, w, d, c).permute(0, 4, 3, 1, 2)
    x = F.conv_transpose3d(x, sd[p + "up.0.weight"], sd[p + "up.0.bias"], stride=dr)
    x = layer_norm_3d(x, sd[p + "up.1.weight"], sd[p + "up.1.bias"])
    return F.conv3d(x, sd[p + "prob.weight"], sd[p + "prob.bias"])


# --------------------------------------------------------------------------------------------------
# S1 + stage
# --------------------------------------------------------------------------------------------------
def stage_forward(features, proj_matrices, depth_values, tmp, position3d, sd, stage_idx, args):
    """cost_volume.py:51-133 (eval mode, depth_type 'ce').  Returns the reference's output dict plus the
    intermediates volume_mean / entropy / vis_weight."""
    p = f"fusions.{stage_idx}."
    G = args["base_ch"][stage_idx] if isinstance(args["base_ch"], (list, tuple)) else args["base_ch"]
    cv = cost_volume(features, proj_matrices, depth_values, sd, p, G)
    if (p + "cost_reg.down.0.weight") in sd:
        logits = costreg_transformer(cv["volume_mean"], position3d, sd, p + "cost_reg.",
                                     args["transformer_config"][stage_idx])
    else:
        logits = costreg_unet(cv["volume_mean"], sd, p + "cost_reg.")
    pre = logits.squeeze(1)
    prob = F.softmax(pre, dim=1)
    depth = torch.sum(F.softmax(pre * tmp, dim=1) * depth_values, 1)
    conf = prob.max(1)[0]
    out = dict(depth=depth, prob_volume=prob, photometric_confidence=conf, depth_values=depth_values,
               prob_volume_pre=pre)
    out.update(cv)
    return out


# --------------------------------------------------------------------------------------------------
# F5-F7: hypothesis scheduling and 3-D positions
# --------------------------------------------------------------------------------------------------
def init_inverse_range(cur_depth, ndepths, H, W):
    """module.py:692-704 (2-D depth_values branch)."""
    dt = cur_depth.dtype
    inv_min = 1.0 / cur_depth[:, 0]
    inv_max = 1.0 / cur_depth[:, -1]
    itv = torch.arange(0, ndepths, dtype=dt).reshape(1, -1, 1, 1).repeat(1, 1, H, W) / (ndepths - 1)
    hypo = inv_max[:, None, None, None] + (inv_min - inv_max)[:, None, None, None] * itv
    return 1.0 / hypo


def upsample2x_align_corners(x, H, W):
    """F.interpolate(x[B,1,D,h,w], [D,H,W], mode='trilinear', align_corners=True) for unchanged D:
    bilinear in (h,w), source index = dst * (in-1)/(out-1)."""
    B, D, h, w = x.shape
    dt = x.dtype

    def axis(n_in, n_out):
        scale = (n_in - 1) / (n_out - 1) if n_out > 1 else 0.0
        src = torch.arange(n_out, dtype=dt) * torch.tensor(scale, dtype=dt)
        i0 = src.floor().long().clamp(max=n_in - 1)
        i1 = (i0 + 1).clamp(max=n_in - 1)
        l1 = src - i0.to(dt)
        return i0, i1, 1 - l1, l1

    y0, y1, wy0, wy1 = axis(h, H)
    x0, x1, wx0, wx1 = axis(w, W)
    top = x[:, :, y0][:, :, :, x0] * wx0 + x[:, :, y0][:, :, :, x1] * wx1
    bot = x[:, :, y1][:, :, :, x0] * wx0 + x[:, :, y1][:, :, :, x1] * wx1
    return top * wy0[:, None] + bot * wy1[:, None]


def schedule_inverse_range(depth, depth_hypo, ndepths, split_itv, H, W):
    """module.py:707-724 (shift=False)."""
    dt = depth.dtype
    last_itv = 1.0 / depth_hypo[:, 2] - 1.0 / depth_hypo[:, 1]
    inv_min = 1 / depth + split_itv * last_itv
    inv_max = 1 / depth - split_itv * last_itv
    itv = torch.arange(0, ndepths, dtype=dt).reshape(1, -1, 1, 1).repeat(1, 1, H // 2, W // 2) / (ndepths - 1)
    hypo = inv_max[:, None] + (inv_min - inv_max)[:, None] * itv
    hypo = upsample2x_align_corners(hypo, H, W)
    return 1.0 / hypo


def get_position_3d(B, H, W, K, depth_values, depth_min, depth_max, hmin, hmax, wmin, wmax):
    """position_encoding.py:138-161 (normalize=True)."""
    D = depth_values.shape[1]
    dt = depth_values.dtype
    y, x = torch.meshgrid([torch.arange(0, H, dtype=dt), torch.arange(0, W, dtype=dt)], indexing="ij")
    xyz = torch.stack((x.reshape(-1), y.reshape(-1), torch.ones(H * W, dtype=dt))).unsqueeze(0).repeat(B, 1, 1)
    xyz = torch.matmul(torch.inverse(K), xyz)
    pos = xyz.unsqueeze(2).repeat(1, 1, D, 1) * depth_values.reshape(B, 1, D, -1)
    if hmin is None or hmax is None or wmin is None or wmax is None:
        wmin, wmax = pos[:, 0].min(), pos[:, 0].max()
        hmin, hmax = pos[:, 1].min(), pos[:, 1].max()
    pos[:, 0] = (pos[:, 0] - wmin) / (wmax - wmin + 1e-5)
    pos[:, 1] = (pos[:, 1] - hmin) / (hmax - hmin + 1e-5)
    pos[:, 2] = (torch.clamp(pos[:, 2], depth_min, depth_max) - depth_min) / (depth_max - depth_min + 1e-5)
    return pos.reshape(B, 3, D, H, W), hmin, hmax, wmin, wmax


# --------------------------------------------------------------------------------------------------
# F1-F4: FMT with pathway
# --------------------------------------------------------------------------------------------------
def pe2d_sine_norm(d_model, H, W, dtype, max_shape=(128, 128)):
    """position_encoding.py:61-74 -> [1,C,H,W]."""
    pe = torch.zeros((d_model, H, W))
    ypos = torch.ones((H, W)).cumsum(0).float().unsqueeze(0) * max_shape[0] / H
    xpos = torch.ones((H, W)).cumsum(1).float().unsqueeze(0) * max_shape[1] / W
    div = torch.exp(torch.arange(0, d_model // 2, 2).float() * (-math.log(10000.0) / (d_model // 2)))[:, None, None]
    pe[0::4] = torch.sin(xpos * div)
    pe[1::4] = torch.cos(xpos * div)
    pe[2::4] = torch.sin(ypos * div)
    pe[3::4] = torch.cos(ypos * div)
    return pe.unsqueeze(0).to(dtype)


def linear_attention(x, key, value, sd, p, nhead):
    """attention.py:261-291."""
    B, N, C = x.shape
    hd = C // nhead
    q = F.linear(x, sd[p + "q_proj.weight"]).reshape(B, N, nhead, hd)
    k = F.linear(key, sd[p + "k_proj.weight"]).reshape(B, N, nhead, hd)
    v = F.linear(value, sd[p + "v_proj.weight"]).reshape(B, N, nhead, hd)
    q = F.elu(q) + 1
    k = F.elu(k) + 1
    KV = torch.einsum("nshd,nshm->nhmd", k, v)
    Z = 1 / (torch.einsum("nlhd,nhd->nlh", q, k.sum(dim=1)) + 1e-6)
    V = torch.einsum("nlhd,nhmd,nlh->nlhm", q, KV, Z).reshape(B, N, C)
    return F.linear(V, sd[p + "proj.weight"], sd[p + "proj.bias"])


def cross_block(x, key, sd, p, nhead):
    """block.py:336-346, pre-norm, pre_norm_query=False (key/value also pass norm1)."""
    C = x.shape[-1]

    def ln(t, n):
        return F.layer_norm(t, (C,), sd[p + n + ".weight"], sd[p + n + ".bias"], 1e-5)

    xn = ln(x, "norm1")
    kn = ln(key, "norm1") if key is not None else xn
    x = x + sd[p + "ls1.gamma"] * linear_attention(xn, kn, kn, sd, p + "attn.", nhead)
    m = F.linear(F.gelu(F.linear(ln(x, "norm2"), sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])),
                 sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    return x + sd[p + "ls2.gamma"] * m


def fmt_with_pathway(features, sd, fmt_cfg, p="FMT_module."):
    """FMT.py:164-206 + FMT.forward :81-137."""
    B, V, C, H, W = features["stage1"].shape
    nhead = fmt_cfg["nhead"]
    names = fmt_cfg["layer_names"]
    dt = features["stage1"].dtype
    pe = pe2d_sine_norm(C, H, W, dt)
    outs = {k: [] for k in ("stage1", "stage2", "stage3", "stage4")}
    ref_list = []
    for vi in range(V):
        x = (features["stage1"][:, vi] + pe).flatten(2).transpose(1, 2)  # n (h w) c
        if vi == 0:
            for i, name in enumerate(names):
                if name == "self":
                    x = cross_block(x, None, sd, f"{p}FMT.layers.{i}.", nhead)
                    ref_list.append(x)
        else:
            for i, name in enumerate(names):
                key = None
                if name == "cross":
                    key = ref_list[i] if len(ref_list) == len(names) else ref_list[i // 2]
                x = cross_block(x, key, sd, f"{p}FMT.layers.{i}.", nhead)
        s1 = x.transpose(1, 2).reshape(B, C, H, W)
        outs["stage1"].append(s1)
        prev = s1
        for k in (1, 2, 3):
            lat = features[f"stage{k + 1}"][:, vi]
            red = F.conv2d(prev, sd[f"{p}dim_reduction_{k}.weight"])
            up = F.interpolate(red, size=lat.shape[-2:], mode="bilinear") + lat
            prev = F.conv2d(up, sd[f"{p}smooth_{k}.weight"], padding=1)
            outs[f"stage{k + 1}"].append(prev)
    return {k: torch.stack(v, dim=1) for k, v in outs.items()}


# --------------------------------------------------------------------------------------------------
# S2: cascade glue
# --------------------------------------------------------------------------------------------------
def hotpath_forward(features, proj_matrices, depth_values, sd, args, tmp=(5.0, 5.0, 5.0, 1.0), run_fmt=True,
                    keep_intermediates=False):
    """DINOv2_mvsformer_model.py:117-179 from the FPN feature pyramid onwards."""
    if run_fmt:
        features = fmt_with_pathway(features, sd, args["FMT_config"])
    ndepths, ratios = args["ndepths"], args["depth_interals_ratio"]
    Bf, _, _, Hs, Ws = features[f"stage{len(ndepths)}"].shape
    prob_maps = torch.zeros(Bf, Hs, Ws, dtype=depth_values.dtype)
    outputs, stage_out = {}, {}
    hmin = hmax = wmin = wmax = None
    for s in range(len(ndepths)):
        pm = proj_matrices[f"stage{s + 1}"]
        f = features[f"stage{s + 1}"]
        B, V, C, H, W = f.shape
        if s == 0:
            ds = init_inverse_range(depth_values, ndepths[s], H, W)
        else:
            ds = schedule_inverse_range(stage_out["depth"], stage_out["depth_values"], ndepths[s], ratios[s], H, W)
        p3d = None
        if args["cost_reg_type"][s] != "Normal" and args.get("use_pe3d", False):
            K = pm[:, 0, 1, :3, :3]
            p3d, hmin, hmax, wmin, wmax = get_position_3d(B, H, W, K, ds, depth_values.min(), depth_values.max(),
                                                          hmin, hmax, wmin, wmax)
        stage_out = stage_forward(f, pm, ds, tmp[s], p3d, sd, s, args)
        if not keep_intermediates:
            for k in ("volume_mean", "entropy", "vis_weight"):
                stage_out.pop(k)
        outputs[f"stage{s + 1}"] = stage_out
        conf = stage_out["photometric_confidence"]
        if conf.shape[1] != Hs or conf.shape[2] != Ws:
            conf = F.interpolate(conf.unsqueeze(1), [Hs, Ws], mode="nearest").squeeze(1)
        prob_maps = prob_maps + conf
        outputs.update(stage_out)
    outputs["refined_depth"] = stage_out["depth"]
    outputs["photometric_confidence"] = prob_maps / len(ndepths)
    outputs["features"] = features
    return outputs


def state_dict_to(sd, dtype):
    return {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
