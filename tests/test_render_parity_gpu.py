"""GPU: the whole path through the reference-shaped API (run_one_iter_of_nerf) against the golden
vectors of the unmodified reference and the live oracle, forward and gradients.

End-to-end tolerance (SURVEY.md section 7.3 items 2-3): the coarse weights steer where the fine
samples land and the last sample's alpha is a step function of sign(sigma), so fp32 evaluation-order
noise is amplified on a few rays.  The acceptance is therefore written against the spread between
the reference's own fp32 and fp64 evaluations: |ours - ref64| <= K * |ref32 - ref64| (+ floor), and
a fraction-of-elements criterion at rtol 1e-4."""
import pytest
import torch

from helpers import CASES, Case, OUT_NAMES, build_models, err_stats, frac_close

pytestmark = pytest.mark.gpu


def run_ours(c: Case, with_grad=False):
    import nerf_pytorch_b200 as nb

    mc, mf, epf, edf = build_models(c)
    rnd = {k: v.cuda() for k, v in c.randoms.items()}
    ctx = torch.enable_grad() if with_grad else torch.no_grad()
    with ctx:
        out = nb.run_one_iter_of_nerf(c.H, c.W, c.focal, mc, mf, c.ro.cuda(), c.rd.cuda(), c.options, mode=c.mode,
                                      encode_position_fn=epf, encode_direction_fn=edf, randoms=rnd)
        loss = None
        if with_grad:
            tgt = c.target.cuda()
            loss = torch.nn.functional.mse_loss(out[0].reshape(-1, 3), tgt)
            if out[3] is not None:
                loss = loss + torch.nn.functional.mse_loss(out[3].reshape(-1, 3), tgt)
            loss.backward()
    return out, loss, mc, mf


@pytest.mark.parametrize("name", CASES)
def test_forward_against_reference_golden(name):
    c = Case(name)
    out, _, _, _ = run_ours(c)
    ref64, _, _, _ = c.oracle(torch.float64)
    for n, got, want, w64 in zip(OUT_NAMES, out, c.outputs, ref64):
        assert (got is None) == (want is None), n
        if want is None:
            continue
        got = got.cpu()
        assert got.shape == want.shape, (n, got.shape, want.shape)
        assert torch.isnan(got).eq(torch.isnan(want)).float().mean() > 0.98, n
        if n.startswith("disp"):
            # disp = 1/(depth/acc) is ill-conditioned on near-empty rays (NaN at acc == 0 in the reference)
            acc = c.outputs[OUT_NAMES.index(n.replace("disp", "acc"))]
            m = (acc > 1e-2) & ~torch.isnan(want)
            assert frac_close(got[m], want[m], rtol=1e-3, atol=1e-5) > 0.97, n
            continue
        spread = (want.double() - w64).abs().max().item()  # what fp32 itself can resolve end to end
        e = (got.double() - w64).abs()
        assert frac_close(got, want, rtol=1e-4, atol=2e-5) > 0.97, (n, err_stats(got, want))
        assert e.median().item() <= 10 * max(spread, 1e-6), (n, e.median().item(), spread)


@pytest.mark.parametrize("name", ["lego_a0_train", "fern_a0_ndc", "a1_skip_lindisp", "a0_noview_coarse_only",
                                  "lego_a0_det_white_val"])
def test_loss_and_gradients_against_oracle(name):
    c = Case(name)
    out, loss, mc, mf = run_ours(c, with_grad=True)
    _, loss64, gc64, gf64 = c.oracle(torch.float64, with_grad=True)
    assert abs(loss.item() - c.loss) <= 2e-3 * abs(c.loss) + 1e-6, (loss.item(), c.loss)
    for tag, model, g64 in (("c", mc, gc64), ("f", mf, gf64)):
        if model is None:
            continue
        tot_num = tot_den = 0.0
        for k, p in model.named_parameters():
            assert p.grad is not None, k
            want = g64[k]
            got = p.grad.double().cpu()
            tot_num += (got - want).pow(2).sum().item()
            tot_den += want.pow(2).sum().item()
        rel = (tot_num / max(tot_den, 1e-300)) ** 0.5
        # whole-gradient relative L2 error; discontinuities (last-sample alpha, resampling) can move a
        # few rays' contribution, hence 1e-2 end-to-end (stage-level tests hold 2e-4)
        assert rel < 1e-2, (name, tag, rel)


def test_validation_mode_shapes_and_mode_quirk():
    import nerf_pytorch_b200 as nb

    c = Case("lego_a0_det_white_val")
    out, _, _, _ = run_ours(c)
    assert out[0].shape == c.ro.shape and out[1].shape == c.ro.shape[:-1] and out[5].shape == c.ro.shape[:-1]


def test_unsupported_inputs_fail_loudly():
    import nerf_pytorch_b200 as nb

    c = Case("lego_a0_train")
    mc, mf, epf, edf = build_models(c)
    with pytest.raises(NotImplementedError):
        nb.run_one_iter_of_nerf(c.H, c.W, c.focal, mc.cpu(), mf, c.ro.cuda(), c.rd.cuda(), c.options,
                                encode_position_fn=epf, encode_direction_fn=edf)
    with pytest.raises(NotImplementedError):
        nb.run_one_iter_of_nerf(c.H, c.W, c.focal, torch.nn.Linear(3, 4).cuda(), None, c.ro.cuda(), c.rd.cuda(),
                                c.options, encode_position_fn=epf, encode_direction_fn=edf)
    with pytest.raises(NotImplementedError):  # CPU rays: no CPU path
        nb.run_one_iter_of_nerf(c.H, c.W, c.focal, mc.cuda(), mf, c.ro, c.rd, c.options,
                                encode_position_fn=epf, encode_direction_fn=edf)


def test_opaque_reference_style_lambda_encoders_are_recognised():
    """The reference passes lambdas (nerf_helpers.py:160-167); they are probed, not rejected."""
    import nerf_pytorch_b200 as nb
    from oracle import nerf_oracle as O

    c = Case("lego_a0_train")
    mc, mf, _, _ = build_models(c)
    epf = lambda x: O.positional_encoding(x, 10, True, True)  # noqa: E731
    edf = lambda x: O.positional_encoding(x, 4, True, True)  # noqa: E731
    rnd = {k: v.cuda() for k, v in c.randoms.items()}
    with torch.no_grad():
        out = nb.run_one_iter_of_nerf(c.H, c.W, c.focal, mc, mf, c.ro.cuda(), c.rd.cuda(), c.options,
                                      encode_position_fn=epf, encode_direction_fn=edf, randoms=rnd)
    assert frac_close(out[3].cpu(), c.outputs[3], rtol=1e-4, atol=2e-5) > 0.97
