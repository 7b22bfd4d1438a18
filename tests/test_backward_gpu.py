"""Gradient parity of the fused backward kernel (MLP dgrad/wgrad on wgmma, table/vector scatter)
with torch autograd through the CPU oracle.  Gradient tiles are bf16 inside the kernel, so the bar is
norm-wise: |g - g_ref| / |g_ref| <= 3e-2 per parameter tensor (and the touched-entry pattern matches)."""
import numpy as np
import pytest
import torch

from helpers import input_batch_of, make_pair, positions_of, synthetic_rays
from oracle import rendering as R

pytestmark = pytest.mark.gpu


def _relnorm(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _oracle_param_list(om):
    ps = []
    for s in om.segments:
        ps += [g for g in s.grids] + [s.vectors]
    return ps + [om.w_sigma, om.w_color]


@pytest.mark.parametrize("segs", [(6,), (6, 6)], ids=["1seg", "2seg"])
@pytest.mark.parametrize("use_saved_features", [True, False, "composed-only"])
def test_field_backward_matches_autograd(cuda, segs, use_saved_features):
    om, m, frames = make_pair(segs)
    for p in om.parameters():
        p.requires_grad_(True)
    b = synthetic_rays(80, 30, frames, ragged=True, seed=11)
    pos, dirs, fr = positions_of(b), b["d"][b["ri"]], b["frames"][b["ri"]]
    n = pos.shape[0]
    g = torch.Generator().manual_seed(5)
    d_sigma = torch.randn(n, generator=g) * 1e-2
    d_rgb = torch.randn(n, 3, generator=g)
    osig, _, orgb = om.forward(pos, dirs, fr)
    ((osig * d_sigma).sum() + (orgb * d_rgb).sum()).backward()

    nat = m.native()
    s = nat.samples_query(pos.to(cuda).contiguous(), dirs.to(cuda).contiguous(), fr.to(cuda).contiguous())
    _, _, _, feat = nat.forward(s, 1, want_geo=False, want_feat=True)
    params = m.hot_parameters()
    grads = [torch.zeros_like(p) for p in params]
    saved = {True: feat, False: None, "composed-only": feat[: n * 32].clone()}[use_saved_features]   # full / re-encode / re-gather
    nat.backward(s, d_sigma.to(cuda), d_rgb.to(cuda).contiguous(), saved, grads)
    torch.cuda.synchronize()

    i = 0
    for si, seg in enumerate(om.segments):
        for k in range(4):
            ref = seg.grids[k].grad.reshape(-1)
            got = grads[i].cpu()
            assert ((got != 0) & (ref == 0)).sum() == 0, "gradient written to an untouched table entry"
            e = _relnorm(got, ref)
            print(f"seg{si} grid{k} relnorm {e:.3e} touched {(ref != 0).sum().item()}")
            assert e < 3e-2
            i += 1
        e = _relnorm(grads[i].cpu(), seg.vectors.grad)
        print(f"seg{si} vectors relnorm {e:.3e}")
        assert e < 3e-2
        i += 1
    ref_sigma = torch.cat([w.grad.reshape(-1) for w in om.w_sigma])
    ref_color = torch.cat([w.grad.reshape(-1) for w in om.w_color])
    es, ec = _relnorm(grads[i].cpu(), ref_sigma), _relnorm(grads[i + 1].cpu(), ref_color)
    print(f"sigma-net relnorm {es:.3e}  colour-net relnorm {ec:.3e}")
    assert es < 3e-2 and ec < 3e-2


@pytest.mark.parametrize("use_saved_features", [True, False])
def test_per_table_backward_equals_single_launch(cuda, use_saved_features):
    """hrf_field_backward == hrf_field_backward_mlp + 4 x hrf_field_backward_tables(k, 1): the schedule the
    data-parallel trainer overlaps with its per-table all-reduces (differences: fp32 atomic ordering only)."""
    _, m, frames = make_pair((6, 6))
    b = synthetic_rays(300, 40, frames, ragged=True, seed=3)
    pos, dirs, fr = positions_of(b), b["d"][b["ri"]], b["frames"][b["ri"]]
    n = pos.shape[0]
    g = torch.Generator().manual_seed(7)
    d_sigma, d_rgb = (torch.randn(n, generator=g) * 1e-2).to(cuda), torch.randn(n, 3, generator=g).to(cuda)
    nat = m.native()
    s = nat.samples_query(pos.to(cuda).contiguous(), dirs.to(cuda).contiguous(), fr.to(cuda).contiguous())
    _, _, _, feat = nat.forward(s, 1, want_geo=False, want_feat=True)
    out = []
    for per_table in (False, True):
        grads = [torch.zeros_like(p) for p in m.hot_parameters()]
        nat.backward(s, d_sigma, d_rgb, feat if use_saved_features else None, grads, per_table=per_table)
        torch.cuda.synchronize()
        out.append(grads)
    for i, (a, b_) in enumerate(zip(*out)):
        assert a.abs().sum() > 0
        e = _relnorm(b_, a)
        assert e < 1e-5, (i, e)


def test_render_autograd_end_to_end(cuda):
    """prune_samples + render + reference loss (trainer.py:205-255) through the module API vs the oracle."""
    from humanrf_b200.volume_rendering import prune_samples, render

    om, m, frames = make_pair((6,), table_std=4.0)
    for p in om.parameters():
        p.requires_grad_(True)
    b = synthetic_rays(150, 48, frames, ragged=True, seed=3)
    ib = input_batch_of(b, cuda)
    nr = ib.num_rays
    # --- pruning (no jitter: is_training=False path so both sides see the same distances)
    with torch.no_grad():
        osig, _ = om.density(positions_of(b), b["frames"][b["ri"]])
    prune_samples(ib, m, is_training=False)
    keep_o = R.prune_mask(osig, b["ri"]).numpy()
    got_t = ib.sample_distances.view(-1).cpu().numpy()
    # the masks may differ only where sigma sits at a threshold within the density tolerance
    exp_t = b["t"].numpy()[keep_o]
    common = np.intersect1d(got_t, exp_t).size
    print("pruned:", got_t.size, "oracle:", exp_t.size, "common:", common)
    assert abs(got_t.size - exp_t.size) <= 0.02 * exp_t.size + 2 and common >= 0.97 * min(got_t.size, exp_t.size)
    assert ib.ray_indices.dtype == torch.int64 and ib.sample_distances.shape[1] == 1
    # --- render + loss on the SAME surviving samples on both sides
    t_k, ri_k = ib.sample_distances.view(-1).cpu(), ib.ray_indices.cpu()
    g = torch.Generator().manual_seed(9)
    bg = torch.rand(nr, 3, generator=g)
    out = render(ib, m, bg.to(cuda), is_training=True)
    loss, _ = R.training_loss(out.color, out.weights_sum, ib.rgba, bg.to(cuda))
    loss.backward()
    pos = b["o"][ri_k] + t_k.unsqueeze(1) * b["d"][ri_k]
    s_o, _, c_o = om.forward(pos, b["d"][ri_k], b["frames"][ri_k])
    col_o, ws_o = R.render(t_k, s_o, c_o, ri_k, nr, bg)
    loss_o, _ = R.training_loss(col_o, ws_o, b["rgba"], bg)
    loss_o.backward()
    print("loss", loss.item(), "oracle", loss_o.item())
    np.testing.assert_allclose(out.color.detach().cpu().numpy(), col_o.detach().numpy(), atol=6e-3)
    np.testing.assert_allclose(out.weights_sum.detach().cpu().numpy(), ws_o.detach().numpy(), atol=6e-3)
    assert abs(loss.item() - loss_o.item()) < 2e-3 * max(1.0, abs(loss_o.item()))
    assert out.color.shape == (nr, 3) and out.weights_sum.shape == (nr, 1)
    refs = [om.segments[0].grids[k].grad.reshape(-1) for k in range(4)] + [om.segments[0].vectors.grad]
    refs += [torch.cat([w.grad.reshape(-1) for w in om.w_sigma]), torch.cat([w.grad.reshape(-1) for w in om.w_color])]
    for p, ref in zip(m.hot_parameters(), refs):
        e = _relnorm(p.grad.cpu(), ref)
        print("param", tuple(p.shape), "relnorm", f"{e:.3e}")
        assert e < 5e-2


def test_adam_step_matches_torch(cuda):
    import ctypes as C

    from humanrf_b200 import _lib as L

    g = torch.Generator().manual_seed(1)
    p0 = torch.randn(10007, generator=g)
    p_ref = p0.clone().to(cuda).requires_grad_(True)
    opt = torch.optim.Adam([p_ref], lr=1e-2, betas=(0.9, 0.99), eps=1e-15)  # run.py:101
    p, m, v = p0.clone().to(cuda), torch.zeros(10007, device=cuda), torch.zeros(10007, device=cuda)
    shadow = torch.empty(10007, dtype=torch.bfloat16, device=cuda)
    for step in range(1, 6):
        grad = (torch.randn(10007, generator=g) * 10 ** float(torch.randint(-6, 1, (1,), generator=g))).to(cuda)
        p_ref.grad = grad.clone()
        opt.step()
        L.check(L.lib().hrf_adam_step(p.data_ptr(), m.data_ptr(), v.data_ptr(), grad.data_ptr(), shadow.data_ptr(), 10007,
                                      1e-2, 0.9, 0.99, 1e-15, step, 1.0, L.stream()))
        np.testing.assert_allclose(p.cpu().numpy(), p_ref.detach().cpu().numpy(), rtol=2e-6, atol=2e-7)
    torch.testing.assert_close(shadow.float(), p.to(torch.bfloat16).float(), rtol=0, atol=0)


def test_camera_embedding_gradients(cuda):
    """render() in training mode with camera_embedding_dim=2: gradients of every parameter incl. the embedding table."""
    from humanrf_b200.volume_rendering import render

    om, m, frames = make_pair((6,), table_std=4.0, cam_emb=2)
    for p in om.parameters():
        p.requires_grad_(True)
    b = synthetic_rays(120, 40, frames, ragged=True, seed=8)
    ib = input_batch_of(b, cuda)
    nr = ib.num_rays
    g = torch.Generator().manual_seed(2)
    bg = torch.rand(nr, 3, generator=g)
    out = render(ib, m, bg.to(cuda), is_training=True)
    loss, _ = R.training_loss(out.color, out.weights_sum, ib.rgba, bg.to(cuda))
    loss.backward()
    pos = positions_of(b)
    s_o, _, c_o = om.forward(pos, b["d"][b["ri"]], b["frames"][b["ri"]], b["cams"][b["ri"]])
    col_o, ws_o = R.render(b["t"], s_o, c_o, b["ri"], nr, bg)
    loss_o, _ = R.training_loss(col_o, ws_o, b["rgba"], bg)
    loss_o.backward()
    assert abs(loss.item() - loss_o.item()) < 2e-3 * max(1.0, abs(loss_o.item()))
    refs = [om.segments[0].grids[k].grad.reshape(-1) for k in range(4)] + [om.segments[0].vectors.grad]
    refs += [torch.cat([w.grad.reshape(-1) for w in om.w_sigma]), torch.cat([w.grad.reshape(-1) for w in om.w_color]),
             om.camera_embeddings.grad]
    for p, ref in zip(m.hot_parameters(), refs):
        e = _relnorm(p.grad.cpu(), ref)
        print("param", tuple(p.shape), "relnorm", f"{e:.3e}")
        assert e < 5e-2
    assert (m.camera_embeddings.weight.grad != 0).any()
