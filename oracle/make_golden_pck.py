"""Generate tests/golden/pck_transfer.npz from the reference's PCK-Transfer code and pin oracle/pck.py against it.

Run where the reference checkout is (GG_REFERENCE_ROOT):  python -m oracle.make_golden_pck
The reference's own ComposedSTN.match_flows, forward_with_flip, transfer_points (both ways) and
applications.pck.pck_transfer(..., device='cpu') run on a seeded similarity -> flow STN (flow 64, supersize 128: the input
downsample runs and S != F).  Its application modules import packages that only the command-line tools use (ray, termcolor,
datasets, utils.vis_tools.helpers); those are stubbed in sys.modules here, and only here.  The oracle and the mirror STN
on the oracle op set must reproduce every result; the reference's results, the key points and the seeds are stored (the
images are rebuilt from their seeds by oracle.make_golden_pck.case_images).
"""
import math
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import opset, refimport  # noqa: E402
from oracle import pck as OP  # noqa: E402
from oracle.make_golden import _save  # noqa: E402

STN_KW = dict(flow_size=64, supersize=128, channel_multiplier=0.25, num_heads=1)
WEIGHT_SEED, WEIGHT_GAIN = 51, 0.6
SIZE, N, P = 128, 6, 10
PERMUTATION = [1, 0, 3, 2, 4, 5, 7, 6, 9, 8]
CASES = [
    # name, iters, padding_mode, transfer_both_ways, num_pairs, visibility column, per-batch threshold flags, image seed
    ("iters1_border_both", 1, "border", True, 10, True, (True, False), 700),
    ("iters3_reflection_oneway", 3, "reflection", False, 9, False, (False, True), 800),
]


def make_stn(get_stn):
    stn = get_stn(["similarity", "flow"], **STN_KW).eval()
    return opset.fill_parameters(stn, WEIGHT_SEED, gain=WEIGHT_GAIN)


def case_images(seed, batch):
    g = torch.Generator().manual_seed(seed * 100 + batch)
    return torch.randn(N, 3, SIZE, SIZE, generator=g), torch.randn(N, 3, SIZE, SIZE, generator=g)


def case_loader(blob, name, image_seed, n_batches=2):
    """The stored batches of a fixture case as the infinite iterator pck_transfer reads."""
    batches = []
    for b in range(n_batches):
        imgsA, imgsB = case_images(image_seed, b)
        d = dict(imgsA=imgsA, imgsB=imgsB, kpsA=blob["%s.b%d.kpsA" % (name, b)], kpsB=blob["%s.b%d.kpsB" % (name, b)])
        if ("%s.b%d.threshB" % (name, b)) in blob:
            for k in ("threshA", "threshB", "scaleA", "scaleB"):
                d[k] = blob["%s.b%d.%s" % (name, b, k)]
        batches.append(d)

    def forever():
        while True:
            for d in batches:
                yield dict(d)
    return forever()


def _stub_modules():
    for name in ("ray", "termcolor", "datasets", "utils.vis_tools", "utils.vis_tools.helpers"):
        if name not in sys.modules:
            mod = types.ModuleType(name)
            mod.__getattr__ = lambda attr, _n=name: (lambda *a, **k: None)
            sys.modules[name] = mod


def _batch(gen, image_seed, b, name, ref_t, iters, padding_mode, visibility, with_thresh):
    """Key points for batch b: random kpsA; kpsB = the reference's own A -> B transfer plus noise of the alpha scales, so
    every alpha sees both outcomes."""
    imgsA, imgsB = case_images(image_seed, b)
    kpsA = torch.rand(N, P, 2, generator=gen) * (SIZE - 17) + 8
    out = {}
    if with_thresh:
        out["threshA"], out["threshB"] = torch.rand(N, generator=gen) * 60 + 30, torch.rand(N, generator=gen) * 60 + 30
        out["scaleA"], out["scaleB"] = torch.rand(N, generator=gen) * 0.5 + 0.75, torch.rand(N, generator=gen) * 0.5 + 0.75
        thrB = out["scaleB"] * out["threshB"]
    else:
        thrB = torch.full((N,), float(SIZE))
    kw = dict(iters=iters, padding_mode=padding_mode)
    _, _, kpsA_m, _, pick = ref_t.match_flows(imgsA, imgsB, kpsA, kpsA.clone(), PERMUTATION, **kw)
    imA = torch.where(pick % 2 == 0, imgsA, imgsA.flip(3))
    imB = torch.where(pick <= 1, imgsB, imgsB.flip(3))
    est = ref_t.transfer_points(imA, imB, kpsA_m, **kw)
    r = torch.rand(N, P, generator=gen) * 0.2 * thrB.view(N, 1)
    ang = torch.rand(N, P, generator=gen) * 2 * math.pi
    kpsB = est + torch.stack([r * torch.cos(ang), r * torch.sin(ang)], -1)
    kpsB[:, :, 0] = torch.where((pick <= 1).view(N, 1), kpsB[:, :, 0], SIZE - 1 - kpsB[:, :, 0])
    if visibility:
        vis = lambda: (torch.rand(N, P, 1, generator=gen) > 0.2).float()
        kpsA, kpsB = torch.cat([kpsA, vis()], -1), torch.cat([kpsB, vis()], -1)
    out["kpsA"], out["kpsB"] = kpsA, kpsB.detach()
    return {"%s.b%d.%s" % (name, b, k): v for k, v in out.items()}


@torch.no_grad()
def gen_pck_transfer():
    refimport.import_reference()
    torch.Tensor.cuda = lambda self, *a, **k: self
    _stub_modules()
    from models.spatial_transformers.spatial_transformer import get_stn
    from applications import pck as ref_pck
    from gangealing_b200.evaluation import pck_transfer
    from gangealing_b200.stn import get_stn as mirror_get_stn
    ref_t = make_stn(get_stn)
    mirror = opset.fill_parameters(mirror_get_stn(["similarity", "flow"], ops=OP.cpu_ops(), **STN_KW).eval(), WEIGHT_SEED,
                                   gain=WEIGHT_GAIN)
    out = {"permutation": torch.tensor(PERMUTATION), "alphas": torch.tensor(OP.ALPHAS)}
    picks_seen = set()
    for ci, (name, iters, padding_mode, both, num_pairs, visibility, thresh_flags, image_seed) in enumerate(CASES):
        kw = dict(iters=iters, padding_mode=padding_mode)
        gen = torch.Generator().manual_seed(9000 + ci)
        for b, with_thresh in enumerate(thresh_flags):
            out.update(_batch(gen, image_seed, b, name, ref_t, iters, padding_mode, visibility, with_thresh))
        for b in range(len(thresh_flags)):
            imgsA, imgsB = case_images(image_seed, b)
            kpsA, kpsB = out["%s.b%d.kpsA" % (name, b)][..., :2], out["%s.b%d.kpsB" % (name, b)][..., :2]
            rA, rB, rpA, rpB, pick = ref_t.match_flows(imgsA, imgsB, kpsA, kpsB, PERMUTATION, **kw)
            oA, oB, opA, opB, opick = OP.match_flows_ref(mirror, imgsA, imgsB, kpsA, kpsB, PERMUTATION, **kw)
            mA, mB, mpA, mpB, mpick = mirror.match_flows(imgsA, imgsB, kpsA, kpsB, PERMUTATION, **kw)
            for got in ((oA, oB, opA, opB, opick), (mA, mB, mpA, mpB, mpick)):
                assert torch.equal(got[4], pick), "%s b%d: picks differ from the reference" % (name, b)
                assert torch.equal(got[0], rA) and torch.equal(got[1], rB), "flipped images differ"
                assert torch.equal(got[2], rpA) and torch.equal(got[3], rpB), "match_flows key points differ"
            picks_seen.update(pick.flatten().tolist())
            estB = ref_t.transfer_points(rA, rB, rpA, **kw)
            estA = ref_t.transfer_points(rB, rA, rpB, **kw)
            nnA = ref_t.congeal_points(rA, rpA, **kw)
            for est, got in ((estB, mirror.transfer_points(rA, rB, rpA, **kw)), (estA, mirror.transfer_points(rB, rA, rpB, **kw))):
                assert (est - got).abs().max() <= 1e-5 * SIZE, "mirror transfer_points deviates"
            assert torch.equal(mirror.congeal_points(rA, rpA, **kw), nnA), "nearest-neighbour indices differ"
            flipped, fw_idx = ref_t.forward_with_flip(imgsA, return_inputs=True, return_flip_indices=True, **kw)[1:]
            _, fl = ref_t(flipped, return_flow=True, **kw)
            from models.losses.loss import total_variation_loss
            scores = -total_variation_loss(fl, reduce_batch=False)
            assert torch.allclose(OP.flow_scores_ref(mirror, imgsA, **kw), scores, rtol=1e-5, atol=1e-7)
            pre = "%s.b%d." % (name, b)
            out.update({pre + "pick": pick.flatten(), pre + "imgsum": torch.stack([rA.double().sum((1, 2, 3)),
                                                                                  rB.double().sum((1, 2, 3))], 1),
                        pre + "pointsA": rpA, pre + "pointsB": rpB, pre + "estB": estB, pre + "estA": estA,
                        pre + "nnA": nnA, pre + "flip_indices": fw_idx.flatten(), pre + "flow_scores": scores})
        perm = PERMUTATION
        pck = ref_pck.pck_transfer(ref_t, case_loader(out, name, image_seed), OP.ALPHAS, num_pairs=num_pairs, device="cpu",
                                   quiet=True, transfer_both_ways=both, permutation=perm, match_flows=True, **kw)
        got = OP.pck_transfer_ref(mirror, case_loader(out, name, image_seed), OP.ALPHAS, num_pairs=num_pairs,
                                  transfer_both_ways=both, permutation=perm, **kw)
        assert torch.equal(got, pck), "%s: oracle PCK %s vs reference %s" % (name, got, pck)
        mine = pck_transfer(mirror, case_loader(out, name, image_seed), OP.ALPHAS, num_pairs=num_pairs, device="cpu",
                            transfer_both_ways=both, permutation=perm, **kw)
        print("%s: reference PCK %s, single-forward evaluator %s" % (name, pck.tolist(), mine.tolist()))
        assert 0 < pck.min() and pck.max() < 1, "every alpha should see both outcomes"
        out[name + ".cfg"] = torch.tensor([iters, {"border": 0, "reflection": 1}[padding_mode], int(both), num_pairs,
                                           int(visibility), image_seed] + [int(f) for f in thresh_flags])
        out[name + ".pck"] = pck
    assert picks_seen == {0, 1, 2, 3}, "fixture must cover every pick value (got %s)" % sorted(picks_seen)
    _save("pck_transfer", **out)


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_pck_transfer()
