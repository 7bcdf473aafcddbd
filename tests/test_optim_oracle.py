"""CPU: the optimiser-tail oracle (oracle/optim_oracle.py) against the golden fixture generated with the reference's own
Queue / get_grad_norm, torch.optim.AdamW(amsgrad) and clip_grad_norm_ (tests/golden/make_golden_optim.py)."""
import os

import torch

import optim_oracle as OO
from conftest import GOLDEN


def load():
    return torch.load(os.path.join(GOLDEN, "optim_steps.pt"), weights_only=False)


def test_oracle_matches_reference_pieces():
    fx = load()
    o = OO.TrainTailOracle(fx["init"])
    for grads, ref in zip(fx["grads"], fx["log"]):
        got = o.step(grads)
        assert abs(got["norm"] - ref["norm"]) <= 1e-5 * ref["norm"]
        assert abs(got["limit"] - ref["limit"]) <= 1e-6 * ref["limit"]
        assert (got["norm"] > got["limit"]) == ref["clipped"]
    assert sum(r["clipped"] for r in fx["log"]) == 2           # the fixture exercises both branches
    for a, b in zip(o.p, fx["params"]):
        assert torch.allclose(a, b, rtol=1e-6, atol=1e-8)
    for a, b in zip(o.ema, fx["ema"]):
        assert torch.allclose(a, b, rtol=1e-6, atol=1e-8)
    for a, b in zip(o.m, fx["exp_avg"]):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6 * float(b.abs().max()))     # sums of +- terms: absolute scale
    for a, b in zip(o.vmax, fx["max_exp_avg_sq"]):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-12)
    assert max(abs(x - y) for x, y in zip(sorted(o.queue.items), fx["history"])) <= 1e-3


def test_queue_is_fifo_of_fifty():
    q = OO.NormQueue(max_len=5)
    for v in range(10):
        q.add(v)
    assert q.items == [9.0, 8.0, 7.0, 6.0, 5.0]


def test_oracle_matches_reference_pieces_past_the_history_window():
    """optim_long.pt (queue_len 1, 3, 50, 120; spikes after the seeded 3000 has left the history; one run without amsgrad)."""
    fx = torch.load(os.path.join(GOLDEN, "optim_long.pt"), weights_only=False)
    assert fx["sizes"] == OO.LONG_SIZES and len(fx["runs"]) == len(OO.LONG_RUNS)
    for r in fx["runs"]:
        init, grads = OO.long_run_grads(r["queue_len"], r["steps"], r["spikes"])
        o = OO.TrainTailOracle(init, amsgrad=r["amsgrad"], queue_len=r["queue_len"])
        for grads_k, ref in zip(grads, r["log"]):
            got = o.step(grads_k)
            assert abs(got["norm"] - ref["norm"]) <= 1e-5 * ref["norm"]
            assert abs(got["limit"] - ref["limit"]) <= 1e-6 * ref["limit"]
            assert (got["norm"] > got["limit"]) == ref["clipped"]
        assert any(l["clipped"] for l in r["log"][r["queue_len"] + 1:])
        arrays = [("params", o.p, 1e-6, 1e-8), ("ema", o.ema, 1e-6, 1e-8)]
        if r["amsgrad"]:
            arrays.append(("max_exp_avg_sq", o.vmax, 1e-5, 1e-12))
        for what, got, rtol, atol in arrays:
            for a, fp in zip(got, r[what]):
                assert torch.allclose(a[OO.fingerprint_index(a.numel())], fp["vals"], rtol=rtol, atol=atol), what
                assert abs(float(a.double().norm()) - fp["norm"]) <= rtol * fp["norm"] + atol, what
        assert len(o.queue.items) == r["queue_len"] and 3000.0 not in o.queue.items
        assert max(abs(x - y) for x, y in zip(sorted(o.queue.items), r["history"])) <= 1e-3
