"""Where a tile of the layer megakernel k_layers_tc spends its time, from the kernel's own clock64 stamps (BDIFF_TIMING=1).

Workload: bench.py's default QM9 forward (128 molecules of 19 atoms, seed-7 weights, tensor mode, the roofline block's
inputs).  The kernel writes, per CTA, {item, t_fetch, t_start, t_end} for its first 16 items and one stamp at every GEMM
phase boundary of one edge tile and one node tile (the first of each kind with item index >= 2).  This tool decodes them
and prints, for edge and node tiles, the median and p90 over CTAs of the dependency wait (t_start - t_fetch), of every
GEMM and epilogue phase, and of the whole tile, next to the k_layers_tc time of profile_forward.
Usage: python tools/layers_phase_profile.py [--config qm9|geom] [--forwards N]"""
import argparse
import os
import subprocess
import sys

os.environ["BDIFF_TIMING"] = "1"      # read when the work buffers are laid out: before the first forward

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "bio-diffusion_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import bdiff  # noqa: E402
import gcpnet_oracle as O  # noqa: E402  (seeded weights only)

# Phases between consecutive stamps, in stamp order (edge_tile_epilogue.inc / node_r4_tile_epilogue.inc: one stamp at the
# tile's start, one before and one after every published GEMM phase, one at the tile's end).  The edge tile's E0 and
# E(k)b run inside their GEMM phases (on the wgmma fragments), so those phases have no stamp between G and E.
EDGE_PHASES = ("T0", "G0+E0", "G1u", "E1a", "G1s+E1b", "G2u", "E2a", "G2s+E2b", "G3u", "E3a", "G3s+E3b", "G4", "sum+E4")
NODE_PHASES = ("T0a", "G1a", "T0v+T0b", "G1b/c", "E1", "G2", "E2", "G3a", "E3a+G4", "G3b", "E3b", "G5|Gp", "E4/E5|Ep")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        pl, sm, smax = (float(x) for x in q.stdout.strip().splitlines()[0].split(","))
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        pl, sm, smax = None, None, None
    return name, pl, sm, smax


def row(label, cyc, mhz):
    cyc = np.asarray(cyc, dtype=np.float64)
    if cyc.size == 0:
        return f"  {label:<10} (no samples)"
    med, p90 = np.median(cyc), np.percentile(cyc, 90)
    us = f"{med / mhz:8.2f} {p90 / mhz:8.2f}" if mhz else "       -        -"
    return f"  {label:<10} {med / 1e3:9.2f} {p90 / 1e3:9.2f}   {us}   n={cyc.size}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="qm9", choices=["qm9", "geom"])
    ap.add_argument("--forwards", type=int, default=5, help="warm-up forwards before the stamped one")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("layers_phase_profile.py needs a CUDA device")
    dev = torch.device("cuda:0")
    dcfg = bdiff.DenoiserConfig.named(args.config)
    net = bdiff.GCPNetDynamicsB200(config=dcfg, mode="tensor")
    net.load_state_dict(O.random_state_dict(O.config_named(args.config), seed=7), strict=True)
    net.to(dev)
    B, A = (128, 19) if args.config == "qm9" else (64, 44)
    bi = torch.repeat_interleave(torch.arange(B), torch.full((B,), A)).to(dev)
    n = bi.shape[0]
    mask = torch.ones(n, dtype=torch.bool, device=dev)
    xh = torch.randn((n, 3 + dcfg.num_h), generator=torch.Generator().manual_seed(3)).to(dev)
    tt = torch.full((n, 1), 0.5, device=dev)
    for _ in range(args.forwards):
        net.denoise(bi, mask, xh, tt, None, B)
    torch.cuda.synchronize()
    kms = []
    for _ in range(5):
        prof, _ = net.profile_forward(bi, mask, xh, tt, None, B)
        kms.append(prof["layers_fused"])
    net.denoise(bi, mask, xh, tt, None, B)            # the stamped forward
    torch.cuda.synchronize()
    name, pl, sm, smax = card()
    dbg = net.debug_tap("dbg").contiguous().view(torch.int64).cpu().numpy().reshape(-1)
    items = dbg[: 256 * 64].reshape(256, 16, 4)
    stamps = dbg[256 * 64:].reshape(256, 2, 32)
    ctas = min(torch.cuda.get_device_properties(0).multi_processor_count, int(np.count_nonzero(items[:, 0, 1])))
    mhz = sm if sm else None

    print(f"card: {name}, power limit {pl} W, SM clock {sm} MHz after the run (max {smax} MHz)")
    print(f"workload: {args.config}, {B} molecules x {A} atoms, tensor mode, {ctas} CTAs")
    print(f"k_layers_tc (profile_forward, mean of 5): {np.mean(kms):.3f} ms  (runs {', '.join(f'{x:.3f}' for x in kms)})")
    print(f"{'':12}{'kcyc med':>9} {'kcyc p90':>9}   {'us med':>8} {'us p90':>8}   (us at the SM clock above)")
    for ty, kind, phases in ((0, "edge", EDGE_PHASES), (1, "node", NODE_PHASES)):
        it = items[:ctas]
        sel = (it[:, :, 1] != 0) & (((it[:, :, 0] >> 30) & 1) == ty)
        wait = (it[:, :, 2] - it[:, :, 1])[sel]
        tile = (it[:, :, 3] - it[:, :, 2])[sel]
        st = stamps[:ctas, ty, : len(phases) + 1]
        ok = np.all(st != 0, axis=1)
        d = np.diff(st[ok], axis=1)
        print(f"{kind} tiles ({int(sel.sum())} items with stamps, {int(ok.sum())} phase-stamped tiles):")
        print(row("dep wait", wait, mhz))
        gsum = np.zeros(d.shape[0])
        esum = np.zeros(d.shape[0])
        for j, ph in enumerate(phases):
            print(row(ph, d[:, j], mhz))
            if ph.startswith("G"):
                gsum += d[:, j]
            else:
                esum += d[:, j]
        print(row("all GEMM", gsum, mhz))
        print(row("all epi", esum, mhz))
        print(row("tile", tile, mhz))


if __name__ == "__main__":
    main()
