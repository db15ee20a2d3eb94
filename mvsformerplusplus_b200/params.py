"""Parameter containers with the reference's state-dict key names and shapes.

The modules built here hold weights only (their ``forward`` is never called): the arithmetic runs in
the CUDA library.  Key names/shapes follow the reference so ``load_state_dict(strict=True)`` of the
hot-path subset of a reference checkpoint works unchanged (reference: test.py:212-220; key inventory
pinned in tests/golden/hotpath_state_dict_keys.txt, produced from models/FMT.py:140-152,
models/cost_volume.py:21-49, models/module.py:367-408,453-504,602-629).
"""
import torch
import torch.nn as nn

from .config import stage_list


class Bag(nn.Module):
    """Named container; never executed."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter container: the hot path runs in the CUDA library")


def _conv_bn2d(cin, cout):
    m = Bag()
    m.conv = nn.Conv2d(cin, cout, 3, padding=1, bias=False)
    m.bn = nn.BatchNorm2d(cout)
    return m


def _conv_bn3d(cin, cout, stride):
    m = Bag()
    m.conv = nn.Conv3d(cin, cout, 3, stride=stride, padding=1, bias=False)
    m.bn = nn.BatchNorm3d(cout)
    return m


def _deconv_bn3d_named(cin, cout, stride, opad):
    m = Bag()
    m.conv = nn.ConvTranspose3d(cin, cout, 3, stride=stride, padding=1, output_padding=opad, bias=False)
    m.bn = nn.BatchNorm3d(cout)
    return m


def _deconv_bn3d_seq(cin, cout, stride, opad):
    return nn.Sequential(nn.ConvTranspose3d(cin, cout, 3, stride=stride, padding=1, output_padding=opad, bias=False),
                         nn.BatchNorm3d(cout), nn.ReLU(inplace=True))


class _LN3D(Bag):
    def __init__(self, c):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c))
        self.bias = nn.Parameter(torch.zeros(c))


def _cross_block(dim, hidden):
    b = Bag()
    b.norm1 = nn.LayerNorm(dim)
    b.attn = Bag()
    b.attn.q_proj = nn.Linear(dim, dim, bias=False)
    b.attn.k_proj = nn.Linear(dim, dim, bias=False)
    b.attn.v_proj = nn.Linear(dim, dim, bias=False)
    b.attn.proj = nn.Linear(dim, dim, bias=True)
    b.ls1 = Bag()
    b.ls1.gamma = nn.Parameter(torch.ones(dim))
    b.norm2 = nn.LayerNorm(dim)
    b.mlp = Bag()
    b.mlp.fc1 = nn.Linear(dim, hidden)
    b.mlp.fc2 = nn.Linear(hidden, dim)
    b.ls2 = Bag()
    b.ls2.gamma = nn.Parameter(torch.ones(dim))
    return b


def build_fmt(fmt_cfg):
    d = fmt_cfg["d_model"]
    bc = fmt_cfg.get("base_channel", 8)
    m = Bag()
    m.FMT = Bag()
    m.FMT.layers = nn.ModuleList([_cross_block(d, 4 * d) for _ in fmt_cfg["layer_names"]])
    iv = fmt_cfg.get("init_values", 1.0)
    for blk in m.FMT.layers:
        nn.init.constant_(blk.ls1.gamma, iv)
        nn.init.constant_(blk.ls2.gamma, iv)
    m.dim_reduction_1 = nn.Conv2d(bc * 8, bc * 4, 1, bias=False)
    m.dim_reduction_2 = nn.Conv2d(bc * 4, bc * 2, 1, bias=False)
    m.dim_reduction_3 = nn.Conv2d(bc * 2, bc, 1, bias=False)
    m.smooth_1 = nn.Conv2d(bc * 4, bc * 4, 3, padding=1, bias=False)
    m.smooth_2 = nn.Conv2d(bc * 2, bc * 2, 3, padding=1, bias=False)
    m.smooth_3 = nn.Conv2d(bc, bc, 3, padding=1, bias=False)
    return m


def _costreg_unet(c, kind):
    """kind 'CostRegNet' (stride 2 in D,H,W, named deconvs, 3^3 prob without bias) or
    'CostRegNet3D' (stride (1,2,2), Sequential deconvs, 1^3 prob with bias)."""
    m = Bag()
    m.kind = kind
    s = 2 if kind == "CostRegNet" else (1, 2, 2)
    m.conv1 = _conv_bn3d(c, 2 * c, s)
    m.conv2 = _conv_bn3d(2 * c, 2 * c, 1)
    m.conv3 = _conv_bn3d(2 * c, 4 * c, s)
    m.conv4 = _conv_bn3d(4 * c, 4 * c, 1)
    m.conv5 = _conv_bn3d(4 * c, 8 * c, s)
    m.conv6 = _conv_bn3d(8 * c, 8 * c, 1)
    if kind == "CostRegNet":
        m.conv7 = _deconv_bn3d_named(8 * c, 4 * c, 2, 1)
        m.conv9 = _deconv_bn3d_named(4 * c, 2 * c, 2, 1)
        m.conv11 = _deconv_bn3d_named(2 * c, c, 2, 1)
        m.prob = nn.Conv3d(c, 1, 3, padding=1, bias=False)
    else:
        m.conv7 = _deconv_bn3d_seq(8 * c, 4 * c, (1, 2, 2), (0, 1, 1))
        m.conv9 = _deconv_bn3d_seq(4 * c, 2 * c, (1, 2, 2), (0, 1, 1))
        m.conv11 = _deconv_bn3d_seq(2 * c, c, (1, 2, 2), (0, 1, 1))
        m.prob = nn.Conv3d(c, 1, 1)
    return m


def _costreg_transformer(c, tc):
    mid = tc["mid_channel"]
    dr = tuple(tc["down_rate"])
    m = Bag()
    m.kind = "PureTransformerCostReg"
    m.pe_proj = nn.Conv3d(c * 3, c, 1, 1, bias=False)
    m.down = nn.Sequential(nn.Conv3d(c, mid, kernel_size=dr, stride=dr), _LN3D(mid))
    layers = []
    for _ in range(tc["layer_num"]):
        b = Bag()
        b.gamma1 = nn.Parameter(torch.tensor(1.0))
        b.gamma2 = nn.Parameter(torch.tensor(1.0))
        b.attn = Bag()
        b.attn.qkv = nn.Linear(mid, 3 * mid, bias=False)
        b.attn.proj = nn.Linear(mid, mid, bias=True)
        b.norm1 = nn.LayerNorm(mid)
        b.ffn = Bag()
        b.ffn.linear1 = nn.Linear(mid, int(mid * tc["mlp_ratio"]))
        b.ffn.linear2 = nn.Linear(int(mid * tc["mlp_ratio"]), mid)
        b.norm2 = nn.LayerNorm(mid)
        layers.append(b)
    m.attention_layers = nn.ModuleList(layers)
    m.up = nn.Sequential(nn.ConvTranspose3d(mid, c, kernel_size=dr, stride=dr), _LN3D(c))
    m.prob = nn.Conv3d(c, 1, 1)
    return m


def build_stage(args, ndepth, stage_idx):
    c = stage_list(args["base_ch"], stage_idx)
    m = Bag()
    m.vis = nn.Sequential(_conv_bn2d(1, 16), _conv_bn2d(16, 16), _conv_bn2d(16, 8), nn.Conv2d(8, 1, 1), nn.Sigmoid())
    t = args.get("cost_reg_type", ["Normal"] * 4)[stage_idx]
    if t == "PureTransformerCostReg":
        m.cost_reg = _costreg_transformer(c, args["transformer_config"][stage_idx])
    elif ndepth <= args.get("model_th", 8):
        m.cost_reg = _costreg_unet(c, "CostRegNet3D")
    else:
        m.cost_reg = _costreg_unet(c, "CostRegNet")
    return m


FPN_CHS = (8, 16, 32, 64)
# FPNEncoder layers (models/module.py:211-224): name, cin, cout, kernel, stride
FPN_ENCODER_LAYERS = (("conv00", 3, 8, 7, 1), ("conv01", 8, 8, 5, 1), ("downsample1", 8, 16, 5, 2),
                      ("conv10", 16, 16, 3, 1), ("conv11", 16, 16, 3, 1), ("downsample2", 16, 32, 5, 2),
                      ("conv20", 32, 32, 3, 1), ("conv21", 32, 32, 3, 1), ("downsample3", 32, 64, 3, 2),
                      ("conv30", 64, 64, 3, 1), ("conv31", 64, 64, 3, 1))


def build_fpn_encoder(m):
    """models/module.py:208-224 (norm_type 'BN'): encoder.<layer>.conv.weight, encoder.<layer>.bn.*"""
    for name, cin, cout, k, _ in FPN_ENCODER_LAYERS:
        b = Bag()
        b.conv = nn.Conv2d(cin, cout, k, padding=(k - 1) // 2, bias=False)
        b.bn = nn.BatchNorm2d(cout)
        setattr(m, name, b)
    return m


def build_fpn_decoder(m):
    """models/module.py:242-255: decoder.out{k}.0 conv (+bias), .1 BatchNorm, inner{k} 1x1 conv with bias"""
    c = FPN_CHS
    m.out0 = nn.Sequential(nn.Conv2d(c[3], c[3], 1), nn.BatchNorm2d(c[3]))
    for k, (cl, co) in enumerate(((c[2], c[2]), (c[1], c[1]), (c[0], c[0])), start=1):
        setattr(m, f"inner{k}", nn.Conv2d(cl, c[3], 1))
        setattr(m, f"out{k}", nn.Sequential(nn.Conv2d(c[3], co, 3, padding=1), nn.BatchNorm2d(co)))
    return m


def build_vit_decoder(m, init_values=1.0, prev_values=0.5):
    """models/module.py:273-313 (CrossVITDecoder, shipped decoder_cfg): self_attn_blocks.{0,1}, cross_attn_blocks.{0,1,2}
    (CrossBlock d 768, mlp 3072), norm_layers.{0,1} (LayerNorm eps 1e-6), prev_values.{0,1} (scalars), and the conv head
    proj / upsampler0 / upsampler1 (.0 conv with bias, .1 BatchNorm, .2 SiLU)."""
    d, ch = 768, 64
    m.self_attn_blocks = nn.ModuleList([_cross_block(d, 4 * d) for _ in range(2)])
    m.cross_attn_blocks = nn.ModuleList([_cross_block(d, 4 * d) for _ in range(3)])
    for blk in list(m.self_attn_blocks) + list(m.cross_attn_blocks):
        nn.init.constant_(blk.ls1.gamma, init_values)
        nn.init.constant_(blk.ls2.gamma, init_values)
    m.norm_layers = nn.ModuleList([nn.LayerNorm(d, eps=1e-6) for _ in range(2)])
    m.prev_values = nn.ParameterList([nn.Parameter(torch.tensor(float(prev_values))) for _ in range(2)])
    m.proj = nn.Sequential(nn.Conv2d(d, ch * 4, 3, stride=1, padding=1), nn.BatchNorm2d(ch * 4), nn.SiLU())
    m.upsampler0 = nn.Sequential(nn.ConvTranspose2d(ch * 4, ch * 2, 4, stride=2, padding=1), nn.BatchNorm2d(ch * 2),
                                 nn.SiLU())
    m.upsampler1 = nn.Sequential(nn.ConvTranspose2d(ch * 2, ch, 4, stride=2, padding=1), nn.BatchNorm2d(ch), nn.SiLU())
    return m


VIT_DEPTH, VIT_DIM, VIT_PATCH, VIT_GRID = 12, 768, 14, 37   # ViT-B/14 at img_size 518: a 37 x 37 pos_embed grid


def build_vit(m, init_values=1.0):
    """models/dino/dinov2.py:43-165 at the shipped vit_base(img_size=518, patch_size=14, block_chunks=0, ffn_layer="mlp"):
    cls_token, pos_embed [1, 1370, 768], mask_token, patch_embed.proj (14 x 14 conv), blocks.{0..11} (norm1, attn.qkv
    with bias, attn.proj, ls1.gamma, norm2, mlp.fc1 / fc2, ls2.gamma; LayerNorm eps 1e-6) and norm."""
    d = VIT_DIM
    m.cls_token = nn.Parameter(torch.zeros(1, 1, d))
    m.pos_embed = nn.Parameter(torch.zeros(1, VIT_GRID * VIT_GRID + 1, d))
    m.patch_embed = Bag()
    m.patch_embed.proj = nn.Conv2d(3, d, VIT_PATCH, stride=VIT_PATCH)
    blocks = []
    for _ in range(VIT_DEPTH):
        b = Bag()
        b.norm1 = nn.LayerNorm(d, eps=1e-6)
        b.attn = Bag()
        b.attn.qkv = nn.Linear(d, 3 * d)
        b.attn.proj = nn.Linear(d, d)
        b.ls1 = Bag()
        b.ls1.gamma = nn.Parameter(init_values * torch.ones(d))
        b.norm2 = nn.LayerNorm(d, eps=1e-6)
        b.mlp = Bag()
        b.mlp.fc1 = nn.Linear(d, 4 * d)
        b.mlp.fc2 = nn.Linear(4 * d, d)
        b.ls2 = Bag()
        b.ls2.gamma = nn.Parameter(init_values * torch.ones(d))
        blocks.append(b)
    m.blocks = nn.ModuleList(blocks)
    m.norm = nn.LayerNorm(d, eps=1e-6)
    m.mask_token = nn.Parameter(torch.zeros(1, d))
    return m


def build_hotpath_params(args):
    root = Bag()
    root.FMT_module = build_fmt(args["FMT_config"])
    root.fusions = nn.ModuleList([build_stage(args, args["ndepths"][i], i) for i in range(len(args["ndepths"]))])
    return root
