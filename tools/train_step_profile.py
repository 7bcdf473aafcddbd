"""Where a training step spends its time: one CUDA event pair around every kernel and cuBLAS GEMM of the training pass
(bdiff_train_timing), summed per operation, for one GEMM precision.  Same batch as bench.py --config geom_train uses
first (64 GEOM molecules, seed 1000).  Usage: python tools/train_step_profile.py [--tf32]"""
import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "bio-diffusion_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import bdiff  # noqa: E402
import gcpnet_oracle as O  # noqa: E402  (seeded weights only)
from bdiff import _lib  # noqa: E402
from bdiff.datasets import GEOM_N_NODES, sample_num_nodes  # noqa: E402
from bdiff.optim import GCDMTrainTail  # noqa: E402


def main():
    dev = torch.device("cuda:0")
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named("geom"))
    net.load_state_dict(O.random_state_dict(O.config_named("geom"), seed=7), strict=True)
    net.to(dev)
    net.flatten_parameters()
    net.set_train_precision("--tf32" in sys.argv)
    opt = GCDMTrainTail(net.parameters())
    tl = bdiff.GCDMTrainLoss(net, GEOM_N_NODES)
    B = 64
    sizes = sample_num_nodes(GEOM_N_NODES, B, seed=1000)
    g = torch.Generator().manual_seed(17)
    bi = torch.repeat_interleave(torch.arange(B), sizes)
    n = int(bi.shape[0])
    x = torch.randn((n, 3), generator=g) * 2.0
    x = x - (torch.zeros((B, 3)).index_add_(0, bi, x) / sizes[:, None].float())[bi]
    one_hot = torch.nn.functional.one_hot(torch.randint(0, 16, (n,), generator=g), 16).float()
    batch = tuple(v.to(dev) for v in (bi, torch.ones(n, dtype=torch.bool), x, one_hot, torch.zeros((n, 0))))

    def step():
        opt.zero_grad()
        loss = tl(*batch, None)[0].mean()
        loss.backward()
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    lib = _lib.load()
    h = net._handle
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    _lib.check(h, lib.bdiff_train_timing(h, st, 1, None, 0), "bdiff_train_timing(on)")
    ev0.record()
    step()
    ev1.record()
    buf = C.create_string_buffer(1 << 16)
    _lib.check(h, lib.bdiff_train_timing(h, st, 0, buf, len(buf)), "bdiff_train_timing(off)")
    torch.cuda.synchronize()
    print(f"# python tools/train_step_profile.py {' '.join(sys.argv[1:])}")
    print(f"# one training step (loss forward + backward + optimiser), {B} GEOM molecules, {n} atoms, "
          f"{int((sizes.long() ** 2).sum())} edges: {ev0.elapsed_time(ev1):.2f} ms on the stream, events included")
    print(buf.value.decode())


if __name__ == "__main__":
    main()
