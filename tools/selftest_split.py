"""GPU: run the split-bf16 wgmma self test for every variant and print the error against an fp64 matmul."""
import ctypes as C
import sys, os
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "bio-diffusion_b200"))
import torch
import bdiff

lib = bdiff.load_library()
g = torch.Generator().manual_seed(0)
a = torch.randn((128, 128), generator=g).cuda()
w = torch.randn((320, 128), generator=g).cuda()
for variant in (0, 2):
    c = torch.zeros((128, 336), device="cuda")
    rc = lib.bdiff_selftest_split(C.c_void_p(torch.cuda.current_stream().cuda_stream), variant, C.c_void_p(a.data_ptr()),
                                  C.c_void_p(w.data_ptr()), C.c_void_p(c.data_ptr()))
    aa = a.double()
    if variant & 2:
        aa = aa[:32].repeat(4, 1)
    ref = aa @ w.double().t()
    ref[:, 288:] = -ref[:, 288:]
    err = (c[:, :320].double() - ref).abs().max().item() / ref.abs().max().item()
    bf = (aa.float().bfloat16().double() @ w.bfloat16().double().t())
    bf[:, 288:] = -bf[:, 288:]
    errbf = (bf - ref).abs().max().item() / ref.abs().max().item()
    ex = c[:, 320:336]
    r = torch.arange(128, device="cuda", dtype=torch.float32)[:, None] * 8 + torch.arange(8, device="cuda")[None, :]
    ok_ex = torch.equal(ex[:, :8], 1000 + r) and torch.equal(ex[:, 8:], r)
    print(f"variant {variant}: rc={rc} rel err vs fp64 = {err:.3e} (plain bf16 would be {errbf:.3e}); exchange ok = {ok_ex}")
