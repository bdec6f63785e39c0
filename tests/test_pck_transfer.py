"""PCK-Transfer evaluation (csrc/pck.cu, ComposedSTN.match_flows, gangealing_b200.evaluation).

CPU: the oracle (oracle/pck.py) and the mirror STN on the oracle op set against the reference's own match_flows,
transfer_points, forward_with_flip and pck_transfer (tests/golden/pck_transfer.npz); the single-forward evaluator against
the reference's 8N composition; a 2-rank gloo run; the C ABI's argument checks; the error behaviour.
GPU: tv_per_sample against float64; pck_transfer end to end against the CPU oracle op set and the fixture; CUDA-graph
replay and run-to-run bit equality.  The kernels of pck_transfer_points are checked stage by stage over their launch plans
in test_points_family_gpu.py.

Comparisons exempt near-ties by one rule (oracle.pck.*_near_ties): a nearest neighbour whose second-best float64 distance
lies within the rounding band of the best, an error within 1e-4 px of a threshold (scaled up where the grids themselves
differ), and a flip pick whose two smallest smoothness sums lie within rounding.  The tests bound the exempt share."""
import pytest
import torch

from conftest import assert_close, load_golden
from oracle import make_golden_pck as G
from oracle import opset
from oracle import pck as OP
from ranks import run_ranks

DEV = "cuda"
CASES = ("iters1_border_both", "iters3_reflection_oneway")


def _cfg(blob, name):
    v = blob[name + ".cfg"].tolist()
    return dict(iters=v[0], padding_mode=("border", "reflection")[v[1]]), bool(v[2]), v[3], v[5]


def _mirror(ops, transforms=("similarity", "flow"), **kw):
    from gangealing_b200.stn import get_stn
    stn_kw = dict(G.STN_KW, **kw)
    return opset.fill_parameters(get_stn(list(transforms), ops=ops, **stn_kw).eval(), G.WEIGHT_SEED, gain=G.WEIGHT_GAIN)


# ------------------------------------------------------------------------------------------------ CPU
def test_oracle_and_mirror_reproduce_the_reference_fixture():
    """Picks, flipped images and match_flows' key points (both quirks) exactly; transferred points to 1e-6 S (a few ulp
    of the pixel coordinate); nearest-neighbour indices exactly; forward_with_flip and the flow scores."""
    blob = load_golden("pck_transfer")
    t = _mirror(OP.cpu_ops())
    perm = blob["permutation"].tolist()
    picks = set()
    with torch.no_grad():
        for name in CASES:
            kw, _, _, seed = _cfg(blob, name)
            for b in range(2):
                p = "%s.b%d." % (name, b)
                imgsA, imgsB = G.case_images(seed, b)
                kpsA, kpsB = blob[p + "kpsA"][..., :2], blob[p + "kpsB"][..., :2]
                for fn in (OP.match_flows_ref, type(t).match_flows):
                    rA, rB, pA, pB, pick = fn(t, imgsA, imgsB, kpsA, kpsB, perm, **kw)
                    assert torch.equal(pick.flatten(), blob[p + "pick"])
                    assert torch.equal(torch.stack([rA.double().sum((1, 2, 3)), rB.double().sum((1, 2, 3))], 1), blob[p + "imgsum"])
                    assert torch.equal(pA, blob[p + "pointsA"]) and torch.equal(pB, blob[p + "pointsB"])
                picks.update(pick.flatten().tolist())
                assert_close(t.transfer_points(rA, rB, pA, **kw), blob[p + "estB"], atol=1e-6 * G.SIZE, what=p + "A->B")
                assert_close(t.transfer_points(rB, rA, pB, **kw), blob[p + "estA"], atol=1e-6 * G.SIZE, what=p + "B->A")
                assert torch.equal(t.congeal_points(rA, pA, **kw), blob[p + "nnA"])
                _, idx = OP.determine_flips_ref(t, imgsA, **kw)
                assert torch.equal(idx.flatten(), blob[p + "flip_indices"])
                assert_close(OP.flow_scores_ref(t, imgsA, **kw), blob[p + "flow_scores"], rtol=1e-5, what="flow scores")
    assert picks == {0, 1, 2, 3}


def test_match_flows_quirks_without_pointsB_and_permutation():
    """pointsB=None returns four values; without a permutation only x is mirrored (x -> S - 1 - x)."""
    from gangealing_b200.stn.transformer import flip_key_points
    pick = torch.tensor([0, 1, 2, 3]).view(4, 1, 1, 1)
    pa = torch.arange(24.).view(4, 3, 2)
    pb = pa + 100
    a, b = flip_key_points(pick, pa, pb, None, 10)
    assert torch.equal(a[:, :, 0], torch.where((pick % 2 == 0).view(4, 1), pa[:, :, 0], 9 - pa[:, :, 0]))
    assert torch.equal(b[:, :, 0], torch.where((pick <= 1).view(4, 1), pb[:, :, 0], 9 - pb[:, :, 0]))
    perm = torch.tensor([2, 0, 1])
    a, b = flip_key_points(pick, pa, pb, perm, 10)
    assert torch.equal(a[0], pa[0]) and torch.equal(b[:, :, 1], pb[:, :, 1])       # pointsB is never relabelled
    assert torch.equal(a[3], torch.stack([9 - pa[3, :, 0], pa[3, :, 1]], -1)[perm][perm])   # pick 3: permuted twice
    a_only, none = flip_key_points(pick, pa, None, perm, 10)
    assert none is None and torch.equal(a_only[2], pa[2])                          # pick 2 without pointsB: untouched


@pytest.mark.parametrize("name", CASES)
def test_pck_transfer_reproduces_the_reference_pck(name):
    """evaluation.pck_transfer (one 4N forward per batch) and the oracle's 8N composition, both on the oracle op set, give
    the reference's PCK values exactly (uneven num_pairs: the last batch is truncated)."""
    from gangealing_b200.evaluation import pck_transfer
    blob = load_golden("pck_transfer")
    kw, both, num_pairs, seed = _cfg(blob, name)
    t = _mirror(OP.cpu_ops())
    perm = blob["permutation"].tolist()
    ref = blob[name + ".pck"]
    got = pck_transfer(t, G.case_loader(blob, name, seed), OP.ALPHAS, num_pairs=num_pairs, device="cpu",
                       transfer_both_ways=both, permutation=perm, **kw)
    assert torch.equal(got, ref), (got, ref)
    got8 = OP.pck_transfer_ref(t, G.case_loader(blob, name, seed), OP.ALPHAS, num_pairs=num_pairs, transfer_both_ways=both,
                               permutation=perm, **kw)
    assert torch.equal(got8, ref)


def test_similarity_only_and_no_flip_inference_match_the_8n_composition():
    """A similarity-only SpatialTransformer (closed-form congeal and uncongeal) and a composed STN with match_flows=False."""
    from gangealing_b200.evaluation import pck_transfer
    blob = load_golden("pck_transfer")
    kw, _, _, seed = _cfg(blob, CASES[0])
    for transforms in (("similarity",), ("similarity", "flow")):
        t = _mirror(OP.cpu_ops(), transforms)
        a = pck_transfer(t, G.case_loader(blob, CASES[0], seed), OP.ALPHAS, num_pairs=11, device="cpu", match_flows=False, **kw)
        b = OP.pck_transfer_ref(t, G.case_loader(blob, CASES[0], seed), OP.ALPHAS, num_pairs=11, match_flows=False, **kw)
        assert torch.equal(a, b), (transforms, a, b)


def test_single_forward_evaluator_equals_the_8n_composition_on_fresh_inputs():
    """New seeds and key points (not the fixture's): counts of pck_transfer_batch vs the reference composition, outside
    the near-tie exemption, with the exempt share bounded."""
    from gangealing_b200.evaluation.pck import pck_transfer_batch, transfer_arguments
    t = _mirror(OP.cpu_ops())
    g = torch.Generator().manual_seed(77)
    n, p = 8, 24
    imgsA, imgsB = torch.randn(n, 3, 128, 128, generator=g), torch.randn(n, 3, 128, 128, generator=g)
    kpsA, kpsB = torch.rand(n, p, 2, generator=g) * 120 + 4, torch.rand(n, p, 2, generator=g) * 120 + 4
    perm = torch.randperm(p, generator=g)
    alphas = torch.tensor([0.3, 0.15, 0.05])
    with torch.no_grad():
        counts, seen = pck_transfer_batch(t, imgsA, imgsB, kpsA, kpsB, alphas, permutation=perm, iters=3)
        args, kwargs, pick, _ = transfer_arguments(t, imgsA, imgsB, kpsA, kpsB, alphas, permutation=perm, iters=3)
        _, est, _ = OP.pck_transfer_points_ref(*args, **kwargs)
        batch = dict(imgsA=imgsA, imgsB=imgsB, kpsA=kpsA, kpsB=kpsB)
        ref = OP.pck_transfer_ref(t, iter([batch]), alphas.tolist(), num_pairs=n, permutation=perm, iters=3)
    near = OP.threshold_near_ties(est, args[1], args[3], alphas)
    assert near.float().mean() <= 0.05
    assert seen == 2 * n * p
    assert (counts.float() / seen - ref).abs().max() * seen <= near.sum()
    assert 0 < counts.min() and counts.max() < seen


def _gloo_worker(rank, world, ret):
    from gangealing_b200.evaluation import pck_transfer
    blob = load_golden("pck_transfer")
    kw, both, _, seed = _cfg(blob, CASES[0])
    t = _mirror(OP.cpu_ops())
    # rank r sees the stored batches from batch r on: an uneven split of 11 pairs (6 + 5)
    loader = G.case_loader(blob, CASES[0], seed)
    for _ in range(rank):
        next(loader)
    got = pck_transfer(t, loader, OP.ALPHAS, num_pairs=11, device="cpu", transfer_both_ways=both,
                       permutation=blob["permutation"].tolist(), **kw)
    if rank == 0:
        ret["pck"] = got.tolist()


@pytest.mark.timeout(600)
def test_two_rank_gloo_run_equals_the_single_process_result():
    from gangealing_b200.evaluation import pck_transfer
    blob = load_golden("pck_transfer")
    kw, both, _, seed = _cfg(blob, CASES[0])
    t = _mirror(OP.cpu_ops())
    # one process over the same pairs: batch 0 (6 pairs) then the first 5 pairs of batch 1
    single = pck_transfer(t, G.case_loader(blob, CASES[0], seed), OP.ALPHAS, num_pairs=11, device="cpu",
                          transfer_both_ways=both, permutation=blob["permutation"].tolist(), **kw)
    assert run_ranks(_gloo_worker, 560)["pck"] == single.tolist()


def test_abi_rejects_bad_arguments():
    from gangealing_b200 import _lib
    dll = _lib.load()
    one = 1   # non-null pointer value: validation must reject these calls before dereferencing anything
    assert dll.gg_tv_per_sample(one, one, 2, 1, 8, None) == -1
    assert b"2 x 2" in dll.gg_last_error()
    assert dll.gg_tv_per_sample(one, None, 2, 8, 8, None) == -1
    assert b"null" in dll.gg_last_error()
    assert dll.gg_tv_per_sample(one, one, 0, 8, 8, None) == -1
    ptrs = [one] * 4 + [one] * 5 + [one, None, one, one, one]        # composed STN: matrix_dst unused

    def call(ptrs, b=2, p=5, a=3, s=128, f=64, gh=64, gw=64):
        return dll.gg_pck_transfer(*ptrs, b, p, a, s, f, gh, gw, None)
    assert call(ptrs, b=0) == -1 and b"positive" in dll.gg_last_error()
    assert call(ptrs, p=0) == -1
    assert call(ptrs, a=0) == -1 and b"alpha" in dll.gg_last_error()
    assert call(ptrs, a=9) == -2 and b"8" in dll.gg_last_error()
    assert call(ptrs, gh=32) == -1 and b"disagrees" in dll.gg_last_error()
    assert call(ptrs, gw=65) == -1
    assert call(ptrs, s=1) == -1
    assert call([None] + ptrs[1:]) == -1 and b"null" in dll.gg_last_error()
    assert call(ptrs[:12] + [None, one]) == -1                                  # composed: identity missing
    sim = ptrs[:11] + [None, None, None]                                        # similarity-only: needs matrix_dst
    assert call(sim) == -1 and b"destination matrix" in dll.gg_last_error()
    assert dll.gg_pck_transfer_workspace(2, 5, 64) == 2 * 5 * 16 + 2 * 64 * 64 * 8
    assert dll.gg_pck_transfer_workspace(2, 5, 0) == 2 * 5 * 16


def test_evaluator_refuses_unsupported_configurations():
    from gangealing_b200.evaluation import flow_scores, pck_transfer
    from gangealing_b200.evaluation.ops import pck_transfer_points, tv_per_sample
    t = _mirror(OP.cpu_ops())
    with pytest.raises(TypeError, match="unsupported"):
        pck_transfer(t, iter([]), 0.1, num_pairs=1, device="cpu", alpha_blend=0.5)
    heads = _mirror(OP.cpu_ops(), num_heads=2)
    with pytest.raises(ValueError, match="num_heads"):
        pck_transfer(heads, iter([]), 0.1, num_pairs=1, device="cpu")
    with pytest.raises(ValueError, match="num_heads"):
        flow_scores(heads, torch.zeros(1, 3, 128, 128))
    sim = _mirror(OP.cpu_ops(), ("similarity",))
    batch = dict(imgsA=torch.zeros(1, 3, 128, 128), imgsB=torch.zeros(1, 3, 128, 128), kpsA=torch.zeros(1, 2, 2),
                 kpsB=torch.zeros(1, 2, 2))
    with pytest.raises(ValueError, match="ComposedSTN"):
        pck_transfer(sim, iter([batch]), 0.1, num_pairs=1, device="cpu")           # flip inference needs residual flows
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        tv_per_sample(torch.zeros(1, 4, 4, 2))
    z = torch.zeros(1, 2, 2)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        pck_transfer_points(z, z, None, torch.ones(1), torch.ones(1), torch.zeros(1, 2, 3), 8, matrix_dst=torch.zeros(1, 2, 3))


def test_flow_score_filter():
    from gangealing_b200.evaluation import filter_dataset, get_high_score_indices
    scores = torch.tensor([-3.0, -1.0, -2.0, -0.5, -4.0])
    assert get_high_score_indices(scores, 0.4) == [1, 3]
    assert list(filter_dataset(list("abcde"), scores, 0.4)) == ["b", "d"]


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 2, 2), (5, 7, 33), (4, 128, 128)], ids=lambda s: "x".join(map(str, s)))
def test_tv_per_sample_vs_float64(shape):
    from gangealing_b200.evaluation.ops import tv_per_sample
    g = torch.Generator().manual_seed(sum(shape))
    flow = torch.randn(*shape, 2, generator=g) * torch.tensor([0.3, 2.0, 0.02]).repeat(shape[0])[:shape[0], None, None, None]
    got = tv_per_sample(flow.to(DEV))
    assert_close(got, OP.tv_per_sample_ref(flow.double()), rtol=2e-6, what="tv_per_sample %s" % (shape,))
    assert torch.equal(got, tv_per_sample(flow.to(DEV)))
    with pytest.raises(RuntimeError, match="2 x 2"):
        tv_per_sample(flow[:, :1].to(DEV))


def _transfer_case(composed, b, p, seed, f=64, s=128):
    """Seeded inputs of one pck_transfer_points call: smooth random grids around the identity, random matrices."""
    g = torch.Generator().manual_seed(seed)
    ang = (torch.rand(b, generator=g) - 0.5) * 1.0
    sc = torch.rand(b, generator=g) * 0.5 + 0.8
    m = torch.stack([sc * torch.cos(ang), -sc * torch.sin(ang), (torch.rand(b, generator=g) - 0.5) * 0.3,
                     sc * torch.sin(ang), sc * torch.cos(ang), (torch.rand(b, generator=g) - 0.5) * 0.3], 1).view(b, 2, 3)
    pts = torch.rand(b, p, 2, generator=g) * (s - 9) + 4
    gt = pts + torch.randn(b, p, 2, generator=g) * 8
    vis = (torch.rand(b, p, generator=g) > 0.25).float()
    thresh = torch.rand(b, generator=g) * 60 + 40
    alphas = torch.tensor([0.1, 0.05, 0.01, 0.2, 0.15])
    kw = dict(matrix_dst=torch.roll(m, 1, 0))
    if composed:
        ident = torch.nn.functional.affine_grid(torch.eye(2, 3)[None], (1, 1, f, f), align_corners=False)
        low = torch.randn(b, 2, 8, 8, generator=g) * 0.06
        delta = torch.nn.functional.interpolate(low, size=(f, f), mode="bicubic", align_corners=False).permute(0, 2, 3, 1)
        grid_dst = torch.roll(delta, 1, 0) + torch.nn.functional.affine_grid(torch.roll(m, 1, 0), (b, 1, f, f), align_corners=False)
        kw = dict(delta_src=delta.contiguous(), identity=ident, grid_dst=grid_dst.contiguous())
    return (pts, gt, vis, thresh, alphas, m, s), kw


@pytest.mark.gpu
@pytest.mark.parametrize("composed", [True, False], ids=["composed", "similarity"])
def test_pck_threshold_is_inclusive(composed):
    """pck.py:155 counts err <= alpha * thresh: transfers that land exactly on their ground truth count at threshold 0."""
    from gangealing_b200.evaluation.ops import pck_transfer_points
    args, kw = _transfer_case(composed, 4, 9, seed=3)
    args = [a.to(DEV) if torch.is_tensor(a) else a for a in args]
    kw = {k: v.to(DEV) for k, v in kw.items()}
    _, est, _ = pck_transfer_points(*args, **kw)
    args[1], args[3] = est, torch.zeros(4, device=DEV)
    counts, again, _ = pck_transfer_points(*args, **kw)
    assert torch.equal(again, est)
    assert counts.tolist() == [int((args[2] != 0).sum())] * args[4].numel()


def _seeded_eval_stn(ops, iters_seed=0, s=256):
    return _mirror(ops, flow_size=128, supersize=s)


def _eval_batch(seed, n=10, p=15, s=256):
    g = torch.Generator().manual_seed(seed)
    imgsA, imgsB = torch.randn(n, 3, s, s, generator=g), torch.randn(n, 3, s, s, generator=g)
    kpsA = torch.rand(n, p, 2, generator=g) * (s - 9) + 4
    kpsB = torch.rand(n, p, 2, generator=g) * (s - 9) + 4
    vis = (torch.rand(n, p, generator=g) > 0.2).float()
    thresh = torch.rand(n, generator=g) * 100 + 60
    return imgsA, imgsB, kpsA, kpsB, vis, thresh, torch.randperm(p, generator=g)


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [1, 3])
def test_pck_transfer_end_to_end_vs_cpu_oracle(iters):
    """S = 256, F = 128: the sm_90a evaluator against the same evaluator on the CPU oracle op set, per point: picks,
    nearest-neighbour indices and estimates outside the exemption, counts within the exempt points."""
    from gangealing_b200.evaluation.pck import transfer_arguments
    from gangealing_b200.evaluation.ops import pck_transfer_points
    tc, tg = _seeded_eval_stn(OP.cpu_ops()), _seeded_eval_stn(None).to(DEV)
    imgsA, imgsB, kpsA, kpsB, vis, thresh, perm = _eval_batch(5 + iters)
    alphas = torch.tensor([1.0, 0.5, 0.2])     # the ground truth here is random: alphas large enough to see both outcomes
    kw = dict(iters=iters, padding_mode="border")
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            ac, kc, pick_c, _ = transfer_arguments(tc, imgsA, imgsB, kpsA, kpsB, alphas, thresh, thresh.flip(0), vis, perm, **kw)
            ag, kg, pick_g, _ = transfer_arguments(tg, imgsA.to(DEV), imgsB.to(DEV), kpsA.to(DEV), kpsB.to(DEV), alphas.to(DEV),
                                                   thresh.to(DEV), thresh.flip(0).to(DEV), vis.to(DEV), perm.to(DEV), **kw)
            _, flows = tc(torch.cat([imgsA, imgsB, imgsA.flip(3), imgsB.flip(3)]), return_flow=True, **kw)
            cc, ec, nc = OP.pck_transfer_points_ref(*ac, **kc)
            cg, eg, ng = pck_transfer_points(*ag, **kg)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    n = imgsA.size(0)
    pair_tie = OP.pick_near_ties(OP.tv_per_sample_ref(flows), 1e-4)
    assert pair_tie.float().mean() <= 0.2
    same = (pick_c.flatten() == pick_g.cpu().flatten())
    assert (same | pair_tie).all()
    ok_rows = torch.cat([same, same])
    q = OP.congeal_query_ref(ac[0].double(), ac[5].double(), ac[6], True)
    qg = OP.congeal_query_ref(ag[0].double().cpu(), ag[5].double().cpu(), ag[6], True)
    shift = ((kg["delta_src"].cpu().double() - kc["delta_src"].double()).abs().max() + (qg - q).abs().max()).item()
    assert shift <= 1e-3
    nn_tie = OP.nn_near_ties(kc["delta_src"].double() + kc["identity"].double(), q, 1e-6, perturbation=shift)
    ok = ok_rows[:, None] & ~nn_tie
    assert ok.float().mean() >= 0.8, ok.float().mean()
    assert torch.equal(ng.cpu()[ok], nc[ok])
    assert_close(eg.cpu()[ok], ec[ok], atol=2e-2, what="end-to-end estimates (px)")
    thr_tie = OP.threshold_near_ties(ec, ac[1], ac[3], alphas, tol=2e-2)
    slack = ((~ok | thr_tie) & (ac[2] != 0)).sum()
    assert ((cg.cpu() - cc).abs() <= slack).all(), (cg, cc, slack)
    assert cc.max() > 0 and cc.min() < (ac[2] != 0).sum()


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_pck_transfer_on_gpu_vs_reference_fixture(name):
    from gangealing_b200.evaluation import pck_transfer
    blob = load_golden("pck_transfer")
    kw, both, num_pairs, seed = _cfg(blob, name)
    t = _mirror(None).to(DEV)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        got = pck_transfer(t, G.case_loader(blob, name, seed), OP.ALPHAS, num_pairs=num_pairs, transfer_both_ways=both,
                           permutation=blob["permutation"].tolist(), **kw)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    visible_total = 2 * num_pairs * G.P if both else num_pairs * G.P
    assert ((got.cpu() - blob[name + ".pck"]).abs() <= 2.0 / visible_total + 1e-7).all(), (got, blob[name + ".pck"])


@pytest.mark.gpu
def test_pck_transfer_batch_graph_replay_and_bitwise_repeatability():
    from gangealing_b200.evaluation import pck_transfer_batch
    t = _seeded_eval_stn(None).to(DEV)
    imgsA, imgsB, kpsA, kpsB, vis, thresh, perm = [x.to(DEV) for x in _eval_batch(3)]
    alphas = torch.tensor([0.1, 0.05, 0.01], device=DEV)
    args = (imgsA, imgsB, kpsA, kpsB, alphas, thresh, thresh.flip(0), vis, perm)
    with torch.no_grad():
        first = [x.clone() for x in pck_transfer_batch(t, *args, iters=3)]
        second = pck_transfer_batch(t, *args, iters=3)
        assert all(torch.equal(a, b) for a, b in zip(first, second))
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            pck_transfer_batch(t, *args, iters=3)
        side.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            captured = pck_transfer_batch(t, *args, iters=3)
        imgsA.copy_(imgsA.flip(0))                  # replay on another batch first, then on the original one
        graph.replay()
        imgsA.copy_(imgsA.flip(0))
        graph.replay()
        torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(captured, first))


@pytest.mark.gpu
def test_error_behaviour_on_the_gpu():
    from gangealing_b200.evaluation import pck_transfer, pck_transfer_batch
    from gangealing_b200.evaluation.ops import pck_transfer_points, tv_per_sample
    t = _mirror(None).to(DEV)
    x = torch.zeros(2, 3, 128, 128, device=DEV)
    k = torch.zeros(2, 4, 2, device=DEV)
    a = torch.tensor([0.1], device=DEV)
    with pytest.raises(TypeError, match="unsupported"):
        pck_transfer_batch(t, x, x, k, k, a, alpha=0.5)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        pck_transfer_points(k, k.cpu(), None, torch.ones(2, device=DEV), a, torch.zeros(2, 2, 3, device=DEV), 128,
                            matrix_dst=torch.zeros(2, 2, 3, device=DEV))
    with pytest.raises(RuntimeError, match="2, 4, 2|cuda|CUDA"):
        tv_per_sample(torch.zeros(2, 4, 4, 2))
    with pytest.raises(RuntimeError, match="flow"):
        tv_per_sample(torch.zeros(2, 4, 4, device=DEV))
    m = torch.zeros(2, 2, 3, device=DEV)
    th = torch.ones(2, device=DEV)
    with pytest.raises(RuntimeError, match="gt"):
        pck_transfer_points(k, k[:, :3], None, th, a, m, 128, matrix_dst=m)
    with pytest.raises(RuntimeError, match="visible"):
        pck_transfer_points(k, k, torch.ones(2, 3, device=DEV), th, a, m, 128, matrix_dst=m)
    with pytest.raises(RuntimeError, match="matrix_dst"):
        pck_transfer_points(k, k, None, th, a, m, 128)
    with pytest.raises(RuntimeError, match="at most 8"):
        pck_transfer_points(k, k, None, th, torch.ones(9, device=DEV), m, 128, matrix_dst=m)
    heads = _mirror(None, num_heads=2).to(DEV)
    with pytest.raises(ValueError, match="num_heads"):
        pck_transfer(heads, iter([]), 0.1, num_pairs=1)
