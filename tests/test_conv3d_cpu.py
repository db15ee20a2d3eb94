"""tests/conv3d_common.py restates how csrc/conv3d_tc.cu tiles a 3x3x3 layer and how csrc/costreg_unet.cu schedules the
nine layers of a U-Net; the GPU tests size their cases from that restatement so that the persistent CTAs loop.  A
retiling of either file fails here, with no GPU, until the restatement follows it."""
import os
import re

from tests import conv3d_common as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _source(name):
    return " ".join(open(os.path.join(ROOT, "mvsformerplusplus_b200", "csrc", name)).read().split())


def test_conv3d_launch_restatement_follows_the_source():
    src = _source("conv3d_tc.cu")
    for line in (
            # geometry of a tile and its shared-memory planes (c3::Geo), weight slabs
            "constexpr int THREADS = 384, MAX_STAGES = 8;", "static constexpr int TW = 8 * NT, TH = 16;",
            "PR = MODE == CONV_S1 ? TH + 2 : TH + 1;", "PC = MODE == CONV_S1 ? TW + 2 : TW + 1;",
            "NSUB = MODE == CONV_S2 ? 4 : 1;", "SUB_BYTES = PR * PC * 16;", "PAIR = (2 * SUB_BYTES + 127) / 128 * 128;",
            "OCT_BYTES = NSUB * PAIR;", "return cout < 16 ? 16 : cout;",
            "return (uint32_t)npad(cout) * (mode == DECONV_S2 ? 1024u : 576u);",
            "int conv3d_tc_kg(int mode, int cin) { return (mode != CONV_S2 && cin >= 16) ? 2 : 1; }",
            "int conv3d_tc_col(int mode, int sd, int cout) { return (mode == CONV_S1 || (mode == CONV_S2 && sd == 1)) "
            "&& c3::npad(cout) <= 32; }",
            # depth taps of an output slice: the units of a tile
            "if (MODE == CONV_S1) id = od + kd - 1; else if (MODE == CONV_S2) id = od * SD + kd - 1;",
            "const int num = od + 1 - kd; if (SD == 1) id = num; else { ok = (num & 1) == 0; id = num >> 1; }",
            "if (ok && id >= 0 && id < ID) { t.kd[t.n] = kd; t.id[t.n] = id; ++t.n; }",
            # launch_mode: tile width, tile count, grid, persistent loop
            "else { OD = a.ID * a.SD; OH = a.IH * 2; OW = a.IW * 2; cells_h = a.IH; cells_w = a.IW; }",
            "const int nts[3] = {4, 2, 1};",
            "const size_t stage = align_up((size_t)a.KG * oct + b_bytes, 128);",
            "if (nt * ncls * NPAD > 256 || 2 * stage + 256 > 227 * 1024) continue;",
            "const long long ntiles = (long long)cdiv(cells_w, 8 * nt) * cdiv(cells_h, 16) * OD;",
            "const double eff = (double)ntiles / (double)(cdiv(ntiles, num_sms) * (long long)num_sms);",
            "if (eff >= 0.85) { best_nt = nt; break; }", "if (eff > best_eff) { best_eff = eff; best_nt = nt; }",
            "const int tiles_w = cdiv(cells_w, 8 * NT), tiles_h = cdiv(cells_h, 16);",
            "const int grid = (int)(ntiles < num_sms ? ntiles : num_sms);",
            "for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) { const int tw = tile % tiles_w, "
            "th = (tile / tiles_w) % tiles_h, od = tile / (tiles_w * tiles_h);",
            "const int U = dt.n * ngroups;",
            # launch_col: resident weights, tile width and depth run
            "const size_t slab = (size_t)NPAD * 1728;", "const int wres = wres_bytes <= 112 * 1024 ? 1 : 0;",
            "if (3 * nt * NPAD > 128) continue;",
            "const size_t stage = align_up((size_t)a.KG * oct + (wres ? 0 : slab), 128);",
            "const size_t fixed = (wres ? wres_bytes : 0) + 256;", "if (ns > c3::MAX_STAGES) ns = c3::MAX_STAGES;",
            "if (ns < 2) continue;", "for (int div = 1; div <= 8; div *= 2) {",
            "if (div > 1 && dc == cdiv(D, div / 2)) continue;",
            "const long long items = (long long)cdiv(OW, 8 * nt) * cdiv(OH, 16) * cdiv(D, dc);",
            "const double halo_w = MODE == CONV_S1 ? (8.0 * nt + 2) / (8.0 * nt) : (16.0 * nt + 1) / (16.0 * nt);",
            "const double halo_d = dc >= D ? 1.0 : (dc + 2.0) / dc;", "const double cost = halo_w * halo_d / eff;",
            "if (cost < best_cost) {",
            "const long long nitems = (long long)tiles_w * tiles_h * cdiv(a.ID, DC);",
            "const int grid = (int)(nitems < num_sms ? nitems : num_sms);",
            "if (a.col) return mode == CONV_S1 ? launch_col<CONV_S1>(a, s) : launch_col<CONV_S2>(a, s);"):
        assert line in src, line
    assert "int NS = (int)((227 * 1024 - 256) / stage);" in src and "int ns = (int)((227 * 1024 - fixed) / stage);" in src
    hdr = _source("conv3d_tc.cuh")
    assert "enum ConvTcMode { CONV_S1 = 0, CONV_S2 = 1, DECONV_S2 = 2 };" in hdr
    assert "enum ConvTcOut { OUT_SPLIT = 0, OUT_F32 = 1, OUT_PROB = 2 };" in hdr


def test_unet_schedule_restatement_follows_the_source():
    src = _source("costreg_unet.cu")
    ch = src[src.index("constexpr int kLayerCh[9][2] = {"):]
    ch = [tuple(int(v) for v in t.split(",")) for t in ch[ch.index("{{") + 2:ch.index("}};")].split("}, {")]
    assert tuple(ch) == C.LAYER_CH
    mode = src[src.index("static const int kLayerMode[9] = {"):]
    mode = [m.strip() for m in mode[mode.index("{") + 1:mode.index("};")].split(",")]
    assert tuple(["CONV_S1", "CONV_S2", "DECONV_S2"].index(m) for m in mode) == C.LAYER_MODE
    assert "const int SD = kind == 0 ? 2 : 1;" in src
    assert "const int D1 = (D - 1) / SD + 1, H1 = H / 2, W1 = W / 2;" in src
    # input extent of every layer launch (conv(l, ..., ID, IH, IW)), the last one in its own block
    ext = {int(l): (d, h, w) for l, d, h, w in re.findall(r"conv\((\d), [^;]*?, (D\d?), (H\d?), (W\d?)\)\)", src)}
    assert ext == {0: ("D", "H", "W"), 1: ("D1", "H1", "W1"), 2: ("D1", "H1", "W1"), 3: ("D2", "H2", "W2"),
                   4: ("D2", "H2", "W2"), 5: ("D3", "H3", "W3"), 6: ("D3", "H3", "W3"), 7: ("D2", "H2", "W2")}
    assert "a.SD = SD; a.ID = D1; a.IH = H1; a.IW = W1;" in src
    assert "if ((rc = launch_conv3d_tc(a, DECONV_S2, OUT_PROB, s))) return rc;" in src
    assert "if ((rc = launch_conv3d_tc(a, DECONV_S2, OUT_F32, s))) return rc;" in src
    ext[8] = ("D1", "H1", "W1")
    for kind, D in ((0, 24), (1, 13)):   # level k: depth (D - 1) / SD + 1 applied k times, H / 2^k, W / 2^k
        depth = [D]
        for _ in range(3):
            depth.append((depth[-1] - 1) // (2 - kind) + 1)
        for l, (m, sd, ci, co, ID, IH, IW, skip, out) in enumerate(C.unet_layers(kind, D, 8 * 17, 8 * 29)):
            k = int(ext[l][0][1:] or 0)
            assert (m, ci, co, sd) == (C.LAYER_MODE[l],) + C.LAYER_CH[l] + (2 - kind,)
            assert (ID, IH, IW) == (depth[k], 8 * 17 >> k, 8 * 29 >> k), l
            assert skip == (l >= 6) and out == (C.OUT_SPLIT if l < 8 else C.OUT_F32 if kind == 0 else C.OUT_PROB)


def test_restated_tile_counts():
    """what the restatement says about an H100 SXM (132 SMs): the last layer of every shipped U-Net runs 864-4080
    tiles, CostRegNet's conv5 / conv6 run 36 (DTU) and 48 (T&T) tiles, and no layer case of the parent suite ran the
    tile kernel with more tiles than CTAs (the largest: 90 tiles of a 32 -> 16 transposed conv)"""
    cov = {(name, st): C.unet_coverage(kind, D, H, W, 132) for name, st, kind, D, H, W in C.stage_shapes()}
    assert sorted(c[8][1]["work"] for c in cov.values()) == [864, 1152, 1728, 2040, 3456, 4080]
    assert [cov["dtu", 2][l][1]["work"] for l in (4, 5)] == [36, 36]
    assert [cov["tt", 2][l][1]["work"] for l in (4, 5)] == [48, 48]
    assert cov["dtu", 4][8][1]["instance"] == (C.DECONV_S2, 4, C.OUT_PROB, 16)
    assert cov["dtu", 2][8][1]["instance"] == (C.DECONV_S2, 4, C.OUT_F32, 16)
    r = C.launch(C.DECONV_S2, 2, 32, 16, 3, 40, 72, 132)
    assert (r["kernel"], r["work"], r["trips"]) == ("tile", 90, (1, 1))
    # the depth-streaming kernel at 64 x 1200: 600 items, depth runs of the whole volume
    r = C.launch(C.CONV_S1, 1, 16, 16, 9, 64, 1200, 132)
    assert (r["kernel"], r["work"], r["dc"], r["trips"]) == ("col", 600, 9, (4, 5))
