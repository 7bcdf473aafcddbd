"""GPU: bdiff.collate.PackedDataset.collate (k_collate_count, k_collate_scatter, k_prepare_context) on the layouts the QM9
fixture of test_gpu_collate.py leaves out — pads 29 .. 200 (one to seven 32-slot warp windows), 5 and 16 atom types,
holes in the present atoms, molecules with no present atom, batches of 1, 8, 9 and 1 037 molecules (one or many CTAs of 8
warps) with repeated and unsorted ids, 1 to 3 conditioning properties over several blocks — against the plain torch
expression of tests/collate_layouts.py, itself checked against the oracle by tests/test_collate_oracle.py: bit-exact.
Then a GEOM-shaped packed batch through the GEOM denoiser against the oracle's forward."""
import pytest
import torch

import collate_layouts as CL

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("num_types", CL.NUM_TYPES)
@pytest.mark.parametrize("pad", CL.PADS)
def test_packed_collation_of_every_layout_is_bit_exact(pad, num_types):
    from bdiff.collate import PackedDataset
    data, norms = CL.padded_dataset(pad, num_types)
    ds = PackedDataset(data, torch.device("cuda"), properties=CL.PROPS)
    for kind, cond in CL.BATCHES.items():
        idx = CL.batch_ids(kind, ds.m)
        ref = CL.packed_reference(data, norms, idx, cond)
        b = ds.collate(idx, conditioning=cond, property_norms=norms)
        assert b.num_graphs == idx.numel() and b.num_nodes == ref["x"].shape[0], kind
        assert torch.equal(b.num_nodes_present.cpu(), ref["counts"]), kind
        assert torch.equal(b.batch.cpu(), ref["batch"]), kind
        assert torch.equal(b.x.cpu(), ref["x"]), kind
        assert torch.equal(b.one_hot.cpu(), ref["one_hot"]), kind
        assert torch.equal(b.charges.cpu(), ref["charges"]), kind
        assert torch.equal(b.props_context.cpu(), ref["context"]), kind
        assert b.mask.all() and torch.equal(b.index.cpu(), idx.unsqueeze(-1)), kind
        if kind == "many":                                   # k_prepare_context over several blocks of 256 entries
            assert b.props_context.numel() > 4 * 256


def test_geom_denoiser_runs_on_a_packed_geom_batch():
    """Pad 181, 16 types, charges: a full 181-atom molecule, one whose only atom is in slot 180, one with holes and a
    dense prefix, collated and run through the GEOM denoiser (parity mode), against the oracle's forward on the same
    rows at the parity bar of 5e-5 of max(1, |ref|)."""
    import bdiff
    import gcpnet_oracle as O
    from bdiff.collate import PackedDataset
    data, norms = CL.padded_dataset(181, 16, num_mols=40, seed=1)
    ds = PackedDataset(data, torch.device("cuda"))
    idx = torch.tensor([CL.FULL, 6, CL.LAST_SLOT_ONLY, 5, 6])
    b = ds.collate(idx)
    ref_b = CL.packed_reference(data, norms, idx, ())
    assert torch.equal(b.batch.cpu(), ref_b["batch"]) and torch.equal(b.x.cpu(), ref_b["x"])
    assert b.num_nodes_present.cpu().tolist()[:3] == [181, int((data["charges"][6] > 0).sum()), 1]
    ocfg = O.config_named("geom")
    sd = O.random_state_dict(ocfg, 4)
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named("geom"), mode="parity")
    net.load_state_dict(sd, strict=True)
    net.cuda()
    _, xc = O.centralize(b.x.cpu(), b.batch.cpu(), b.mask.cpu(), b.num_graphs)
    xh = torch.cat((xc, b.one_hot.cpu()), -1).cuda()             # geom: 16 atom types, no charges in the features
    g = torch.Generator().manual_seed(2)
    t = torch.rand((b.num_graphs, 1), generator=g)[b.batch.cpu()].cuda()
    with torch.no_grad():
        _, out = net(b, xh, t)
    ref = O.denoiser_forward(sd, ocfg, b.batch.cpu(), b.mask.cpu(), xh.cpu(), t.cpu())
    assert torch.isfinite(out).all()
    assert (out.cpu() - ref).abs().max().item() <= 5e-5 * max(1.0, ref.abs().max().item())
