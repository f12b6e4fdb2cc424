"""CPU: the float64 appearance-code gradient (tests/appear64.py on oracle/fused64.py) -- per sample (code_grad), per ray (ray_sum) --
against torch float64 autograd."""
import numpy as np
import pytest
import torch

from appear64 import code_grad, ray_sum, step_code_grads
from oracle import fused64, lotd as olotd, nets as onets

CFG16 = olotd.gen_ngp_cfg(log2_hashmap_size=14)


def _ref(n_appear, seed):
    g = torch.Generator().manual_seed(seed)
    meta = olotd.LoDMeta(3, **CFG16)
    table = (torch.rand(meta.n_params, generator=g) * 2 - 1) * 0.5
    lin = lambda o, i: onets.kaiming_linear(g, o, i)
    ws = [*lin(64, 32), *lin(1, 64), *lin(64, 54 + n_appear), *lin(64, 64), *lin(3, 64)]
    return fused64.Fused64(table, CFG16, *ws, rounding=False)


@pytest.mark.parametrize("n_appear", [1, 4, 8])
def test_per_sample_code_gradient_is_autograd_of_the_radiance_head(n_appear):
    ref = _ref(n_appear, seed=3 + n_appear)
    g = torch.Generator().manual_seed(n_appear)
    n = 300
    x = (torch.rand(n, 3, generator=g) * 1.9 - 0.95).numpy()
    v = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).numpy()
    ha = (torch.randn(n, n_appear, generator=g) * 0.5).numpy()
    g_rgb = torch.randn(n, 3, generator=g).double()
    fwd = ref.color_forward(x, v, ha)
    # the radiance head of color_forward in torch: X = [x | SH | n | h | h_appear] with everything but the codes held fixed
    ha_t = torch.tensor(ha, dtype=torch.float64, requires_grad=True)
    X = torch.cat([torch.from_numpy(fwd["X"][:, :54]), ha_t], -1)
    t = lambda a: torch.from_numpy(a)
    Y1 = torch.relu(X @ t(ref.R1).T + t(ref.rb1))
    Y2 = torch.relu(Y1 @ t(ref.R2).T + t(ref.rb2))
    rgb = torch.sigmoid(Y2 @ t(ref.R3).T + t(ref.rb3))
    np.testing.assert_allclose(rgb.detach().numpy(), fwd["rgb"], rtol=1e-12, atol=1e-14)     # the same head
    want = torch.autograd.grad((rgb * g_rgb).sum(), ha_t)[0].numpy()
    got = code_grad(ref, fwd, g_rgb.numpy())
    assert got.shape == (n, n_appear)
    assert np.abs(want).max() > 0
    np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-14 * np.abs(want).max())


def test_per_ray_sum_is_index_add():
    g = torch.Generator().manual_seed(5)
    rows = torch.randn(1000, 4, generator=g, dtype=torch.float64)
    ray = torch.sort(torch.randint(0, 300, (1000,), generator=g))[0]
    ray[500:520] = ray[499]                         # a long run
    want = torch.zeros(310, 4, dtype=torch.float64).index_add_(0, ray, rows).numpy()
    got = ray_sum(rows.numpy(), ray.numpy(), 310)
    np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-13)
    hit = np.zeros(310, bool)
    hit[ray.numpy()] = True
    assert (got[~hit] == 0).all() and (~hit).sum() > 10          # rays without a sample: exactly zero


def test_step_replay_code_gradient_is_autograd_of_the_composited_rgb():
    """step_code_grads (oracle/step64.py's step, unrounded) against torch float64 autograd of sum(g_rgb . rgb_volume) with respect to
    the rays' codes, on the decisions of tests/test_step64_oracle.py (early stops, rays that keep nothing, long packs)"""
    import test_step64_oracle as so
    from oracle import neus64, step64
    _, ref, dec, inv_s, g = so._case()
    got = step_code_grads(ref, dec, inv_s, **g)
    o, d, t1, pinfo, kept, kpi = dec["o"], dec["d"], dec["t1"], dec["pinfo"], dec["kept"], dec["kept_pinfo"]
    R, K = pinfo.shape[0], kept.shape[0]
    ray_b, ray_k = neus64.pack_of(pinfo, t1.shape[0]), neus64.pack_of(kpi, K)
    alpha, _ = neus64.neus_alpha(ref.sdf(step64.points(o[ray_b], d[ray_b], t1)), pinfo, float(np.float32(inv_s)))
    _, w = neus64.transmittance(alpha[kept], dec["vis_fwd"], kpi)
    fwd = ref.color_forward(step64.points(o[ray_k], d[ray_k], dec["t_kept"]), dec["view"][ray_k], dec["h_appear"][ray_k])
    ha_t = torch.tensor(dec["h_appear"], dtype=torch.float64, requires_grad=True)
    X = torch.cat([torch.from_numpy(fwd["X"][:, :54]), ha_t[torch.from_numpy(ray_k)]], -1)
    t = lambda a: torch.from_numpy(a)
    rgb = torch.sigmoid(torch.relu(torch.relu(X @ t(ref.R1).T + t(ref.rb1)) @ t(ref.R2).T + t(ref.rb2)) @ t(ref.R3).T + t(ref.rb3))
    C = torch.zeros(R, 3, dtype=torch.float64).index_add(0, torch.from_numpy(ray_k), t(np.asarray(w, np.float64))[:, None] * rgb)
    want = torch.autograd.grad((C * t(g["g_rgb"])).sum(), ha_t)[0].numpy()
    assert got.shape == want.shape and np.abs(want).max() > 0
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-12 * np.abs(want).max())
    assert (got[kpi[:, 1] == 0] == 0).all()
