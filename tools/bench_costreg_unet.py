"""U-Net cost regularisers of stages 2-4 (CostRegNet D=16, CostRegNet3D D=8 and D=4; models/module.py:367-504) on
cuda:0 at the sizes one depth map runs them, per U-Net and per conv layer.

  * per U-Net: median of --reps CUDA-event timings of one mvsf_costreg_unet_forward (after --warmup calls);
  * per layer: a separate torch.profiler run (CUDA activity only) over --prof-reps forwards; kernels are assigned to
    layers by launch order (split_hi_lo_f16, conv1 .. conv6, conv7 / conv9 / conv11 transposed, [prob3]), median per launch
    over the forwards whose kernels the trace recorded completely.

Next to each layer time it prints what the layer's kernel ISSUES to the tensor cores (the hi/lo split products - 2 MMA
variants for 8-channel groups, 3 for 16-channel groups - and the padding of N to NPAD = max(Cout, 16) included; the
transposed convs issue all 16 (shift, class) weight blocks of which 9 are taps; the depth-streaming convs issue the
3*NPAD-wide product for every input slice of a depth run, taken here as the whole depth) and the algorithmic HBM bytes
(fp16 hi|lo input read once, output and skip tensors once, packed weights once), and the share of the two bounds
those give on an H100 SXM data sheet (989 TFLOP/s dense FP16, 3.35 TB/s HBM3; both for a card allowed 700 W).

  python tools/bench_costreg_unet.py [--workload dtu|tt] [--reps 20] [--warmup 3] [--prof-reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mvsformerplusplus_b200 import packing, synth  # noqa: E402
from mvsformerplusplus_b200.config import default_args  # noqa: E402
from mvsformerplusplus_b200.params import build_hotpath_params  # noqa: E402

WORKLOADS = {"dtu": (1152, 1536), "tt": (1088, 1920)}
STAGES = ((2, 1, 16, 4), (3, 2, 8, 2), (4, 3, 4, 1))   # (stage, fusions index, D, H/W divisor)
PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35
CH = ((8, 16), (16, 16), (16, 32), (32, 32), (32, 64), (64, 64), (64, 32), (32, 16), (16, 8))
MODE = (1, 0, 1, 0, 1, 0, 2, 2, 2)   # conv3d_tc.cuh: CONV_S1 = 0, CONV_S2 = 1, DECONV_S2 = 2
NAMES = ("conv1", "conv2", "conv3", "conv4", "conv5", "conv6", "conv7", "conv9", "conv11")


def depth_taps(mode, od, sd, idepth):
    """number of depth taps of output slice od (conv3d_tc.cu depth_taps)"""
    n = 0
    for kd in range(3):
        if mode == 0:
            i, ok = od + kd - 1, True
        elif mode == 1:
            i, ok = od * sd + kd - 1, True
        else:
            num = od + 1 - kd
            ok = sd == 1 or num % 2 == 0
            i = num // sd
        n += ok and 0 <= i < idepth
    return n


def layer_table(kind, D, H, W):
    """per conv layer: shapes, tensor FLOPs issued and algorithmic HBM bytes"""
    sd = 2 if kind == 0 else 1
    dims = [(D, H, W)]
    for _ in range(3):
        d, h, w = dims[-1]
        dims.append(((d - 1) // sd + 1, h // 2, w // 2))
    ins = [dims[0], dims[1], dims[1], dims[2], dims[2], dims[3], dims[3], dims[2], dims[1]]
    rows = []
    for l in range(9):
        cin, cout = CH[l]
        mode = MODE[l]
        idp, ih, iw = ins[l]
        if mode == 0:
            od, oh, ow = idp, ih, iw
        elif mode == 1:
            od, oh, ow = (idp - 1) // sd + 1, (ih - 1) // 2 + 1, (iw - 1) // 2 + 1
        else:
            od, oh, ow = idp * sd, 2 * ih, 2 * iw
        npad = max(cout, 16)
        kg = 2 if mode != 1 and cin >= 16 else 1
        groups, nv = cin // 8 // kg, (3 if kg == 2 else 2)
        per_mma = 2 * 64 * 16 * npad   # FLOPs of one m64 x N = NPAD x k16 product
        col = (mode == 0 or (mode == 1 and sd == 1)) and npad <= 32
        if col:        # one 3*NPAD product per (input slice, group, tap, variant) and 64 cells
            flop = idp * oh * ow / 64 * groups * 9 * nv * 3 * per_mma
        elif mode == 2:  # per input cell and depth tap: 4 shifts x 4 class blocks
            flop = sum(depth_taps(2, o, sd, idp) for o in range(od)) * ih * iw / 64 * groups * 4 * nv * 4 * per_mma
        else:
            flop = sum(depth_taps(mode, o, sd, idp) for o in range(od)) * oh * ow / 64 * groups * 9 * nv * per_mma
        nin, nout = idp * ih * iw * cin, od * oh * ow * cout
        last = l == 8
        out_bytes = (od * oh * ow * 4 if kind == 1 else nout * 4) if last else nout * 4
        skip_bytes = nout * 4 if l >= 6 else 0
        w_bytes = 27 * cin * npad * 2 * 2
        rows.append({"layer": NAMES[l], "mode": ("s1", "s2", "deconv")[mode] + ("_col" if col else ""),
                     "cin": cin, "cout": cout, "in": [idp, ih, iw], "out": [od, oh, ow],
                     "gflop_issued": flop / 1e9, "mb_hbm": (nin * 4 + out_bytes + skip_bytes + w_bytes) / 1e6})
    return rows


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return [s.strip() for s in q.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="dtu", choices=sorted(WORKLOADS))
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--prof-reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_costreg_unet: no CUDA device (timings are only taken on the GPU)")
    from mvsformerplusplus_b200 import _lib
    from mvsformerplusplus_b200.hotpath import pack_unet_tc
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    sd = synth.randomize_state_dict(build_hotpath_params(default_args()).eval(), seed=13)
    H0, W0 = WORKLOADS[a.workload]
    name, power, sm_clock = card()
    res = {"bench": "costreg_unet", "workload": a.workload, "device": name, "power_limit": power, "max_sm_clock": sm_clock,
           "reps": a.reps, "warmup": a.warmup, "prof_reps": a.prof_reps, "unets": []}
    total_ms = 0.0
    for stage, fi, D, div in STAGES:
        H, W = H0 // div, W0 // div
        kind, conv, small = packing.pack_costreg_unet(sd, f"fusions.{fi}.cost_reg.")
        small_d, tc = small.to(dev), pack_unet_tc(kind, conv.to(dev))
        ws = _lib.workspace("mvsf_costreg_unet_workspace_bytes", kind, 8, D, H, W, device=dev)
        vol = (torch.randn(D, H, W, 8, generator=torch.Generator().manual_seed(stage)) * 0.5).to(dev)
        logits = torch.empty(D, H, W, device=dev)

        def fwd():
            _lib.call("mvsf_costreg_unet_forward", kind, vol, small_d, tc, logits, ws, ws.numel() * 4, 8, D, H, W)

        for _ in range(a.warmup):
            fwd()
        torch.cuda.synchronize()
        ms = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fwd()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        ms.sort()
        med = ms[len(ms) // 2]
        total_ms += med

        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.prof_reps):
                fwd()
            torch.cuda.synchronize()
        kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                       and "memcpy" not in e.name.lower() and "memset" not in e.name.lower()),
                      key=lambda e: e.time_range.start)
        # one forward = split_hi_lo_f16, 9 convs[, prob3]; the trace can miss a kernel record, so only complete forwards count
        fwds = []
        for e in kern:
            if "split_hi_lo_f16" in e.name:
                fwds.append([])
            if fwds:
                fwds[-1].append(e)
        per_fwd = 10 + (kind == 0)
        fwds = [f for f in fwds if len(f) == per_fwd]
        assert fwds, f"no complete forward among {len(kern)} kernel records"
        rows = layer_table(kind, D, H, W)
        layers, li = [], 0
        for k in range(per_fwd):
            times = sorted(f[k].time_range.elapsed_us() / 1e3 for f in fwds)
            t = times[len(times) // 2]
            kname = fwds[0][k].name
            if "conv3d_" in kname:
                row = dict(rows[li])
                li += 1
                row["kernel"] = kname.split("(")[0].replace("void ", "").replace("mvsf::", "")
                row["ms"] = round(t, 4)
                t_flop, t_hbm = row["gflop_issued"] / PEAK_TFLOPS, row["mb_hbm"] / PEAK_TBS / 1e6 * 1e3
                row["share_tensor_bound"] = round(t_flop / t, 3)
                row["share_hbm_bound"] = round(t_hbm / t, 3)
                row["gflop_issued"] = round(row["gflop_issued"], 2)
                row["mb_hbm"] = round(row["mb_hbm"], 1)
            else:
                row = {"layer": "-", "kernel": kname.split("(")[0].replace("void ", "").replace("mvsf::", ""), "ms": round(t, 4)}
            layers.append(row)
        assert li == 9, f"expected 9 conv launches per forward, saw {li}"
        res["unets"].append({"stage": stage, "kind": ("CostRegNet", "CostRegNet3D")[kind], "D": D, "H": H, "W": W,
                             "ms_median": round(med, 4), "ms_min": round(ms[0], 4), "ms_max": round(ms[-1], 4),
                             "profiled_forwards": len(fwds), "launches": layers})
        del ws, vol, logits, small_d, tc
        torch.cuda.empty_cache()
    res["ms_total_median"] = round(total_ms, 4)

    print(f"# {name}, power limit {power}, max SM clock {sm_clock}; workload {a.workload}")
    for u in res["unets"]:
        print(f"## stage {u['stage']} {u['kind']} D={u['D']} {u['H']}x{u['W']}: {u['ms_median']:.3f} ms "
              f"(median of {a.reps}, min {u['ms_min']:.3f}, max {u['ms_max']:.3f})")
        print("| layer | kernel | ms | GFLOP issued | tensor-bound share | MB HBM | HBM-bound share |")
        print("|---|---|---|---|---|---|---|")
        for r in u["launches"]:
            if r["layer"] == "-":
                print(f"| - | {r['kernel']} | {r['ms']:.3f} | | | | |")
            else:
                print(f"| {r['layer']} | {r['kernel']} | {r['ms']:.3f} | {r['gflop_issued']:.1f} | {r['share_tensor_bound']:.2f} "
                      f"| {r['mb_hbm']:.0f} | {r['share_hbm_bound']:.2f} |")
    print(f"## all three U-Nets: {res['ms_total_median']:.3f} ms")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
