"""Geometry-only NeuS models (`radiance_cfg=False`, the reference's `radiance_cfg: null`, e.g. the LiDAR-only StreetSurf configuration):
state-dict keys, strict loading, the adapter's mapping and the refusals -- everything that needs no GPU."""
import pytest
import torch

from neuralsim_b200.fields import LoTDNeuSModel


def _model(radiance_cfg):
    torch.manual_seed(0)
    return LoTDNeuSModel(surface_cfg=dict(bounding_size=2.0), radiance_cfg=radiance_cfg, var_ctrl_cfg=dict(ln_inv_s_init=0.3),
                         accel_cfg=dict(resolution=[8, 8, 8], update_from_samples_cfg=None))


def test_geometry_only_model_has_no_radiance_net():
    m = _model(False)
    assert m.radiance_net is None
    assert (m.use_view_dirs, m.use_nablas, m.use_h_appear) == (False, False, False)
    assert not any(k.startswith("radiance_net.") for k, _ in m.named_parameters())
    assert not any(k.startswith("radiance_net.") for k in m.state_dict())
    assert not m._color_fusable()


def test_geometry_only_keys_are_the_colour_model_keys_without_the_radiance_net():
    geo, col = set(_model(False).state_dict()), set(_model(dict(n_appear_embedding=4)).state_dict())
    assert geo == {k for k in col if not k.startswith("radiance_net.")}
    assert {k.split(".")[0] for k in geo} == {k.split(".")[0] for k in col} - {"radiance_net"}
    assert "ctrl_var.ln_inv_s" in geo and any(k.startswith("accel.occ.") for k in geo)


def test_geometry_only_strict_load_of_its_own_state():
    a, b = _model(False), _model(False)
    with torch.no_grad():
        a.implicit_surface.decoder.layers[0].weight.add_(1.0)
    sd = a.state_dict()
    res = b.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert torch.equal(b.implicit_surface.decoder.layers[0].weight, a.implicit_surface.decoder.layers[0].weight)
    with pytest.raises(RuntimeError):            # a colour checkpoint has keys a geometry-only model lacks
        b.load_state_dict(_model(None).state_dict(), strict=True)


def test_radiance_cfg_none_still_builds_the_default_radiance_net():
    m = _model(None)
    assert m.radiance_net is not None and m.use_view_dirs and m.use_nablas and not m.use_h_appear


def test_geometry_only_forward_refuses_rgb():
    m = _model(False)
    with pytest.raises(RuntimeError, match="no radiance net"):
        m.forward(torch.zeros(4, 3), with_rgb=True)


class _Stub:
    pass


def test_describe_maps_a_missing_radiance_net_to_false():
    from neuralsim_b200.adapter import describe
    src = _model(False)
    ref = _Stub()                    # only the attributes the reference's LoTDNeuS objects have
    ref.implicit_surface, ref.radiance_net, ref.ctrl_var, ref.accel, ref.space = src.implicit_surface, None, src.ctrl_var, src.accel, src.space
    ref.ray_query_cfg = dict(src.ray_query_cfg)
    cfg = describe(ref)
    assert cfg["radiance_cfg"] is False
    ref.radiance_net = _model(dict(n_appear_embedding=4)).radiance_net
    assert describe(ref)["radiance_cfg"]["n_appear_embedding"] == 4
