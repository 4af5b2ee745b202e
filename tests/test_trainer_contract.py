"""The contract between the native models and the trainer seam (``arena.ArenaModule``), checked on the host: every parameter
sits in exactly one of a model's ``arenas()``, ``dp`` wires one bucket reducer per ``exchanges()`` site and ``comm`` and takes
them off again, and the trainer writes nothing onto the model."""
import json
import os

import pytest
import torch

import cflearn_b200  # noqa: F401
from cflearn_b200 import dp, registry
from cflearn_b200.ddpm import DDPMB200
from cflearn_b200.optim import ArenaAdam
from cflearn_b200.trainer import B200TrainStep

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class _Comm:
    """Stands in for a ``dp.NativeComm`` of a two-rank job (nothing here launches a collective)."""

    world = 2
    ctas = 0


def _classifier():
    return registry.build_module("cv_clf", config=dict(in_channels=3, num_classes=10, img_size=32, latent_dim=128, encoder="vit",
                                                       encoder_config=dict(patch_size=16, num_layers=2)))


def _vit_encoder():  # CLIP's vision options: output_projection and embedding_norm
    return registry.build_module("encoders.vit", config=dict(
        img_size=64, patch_size=32, in_channels=3, latent_dim=128, to_patches_config={"bias": False}, num_layers=2,
        norm_kwargs={"eps": 1e-5}, embedding_norm=torch.nn.LayerNorm(128, 1e-5), attention_kwargs={"num_heads": 2},
        feedforward_kwargs={"activation": "quick_gelu"}, norm_after_head=True, output_dim=64))


def _tet_encoder():
    return registry.build_module("tet", config=dict(latent_dim=128, context_length=12, use_triu_attn_mask=True, num_layers=2,
                                                    attention_kwargs={"num_heads": 2}))


def _clip():
    return registry.build_module("clip", config=dict(img_size=64, latent_dim=64, vision_latent_dim=128, vision_patch_size=32,
                                                     vision_num_heads=2, vision_num_layers=1, vocab_size=512, context_length=16,
                                                     text_latent_dim=128, text_num_heads=2, text_num_layers=2))


def _ddpm():
    cfg = json.load(open(os.path.join(GOLDEN, "unet_small64_state_dict_keys.json")))["config"]
    cfg = {k: tuple(v) if isinstance(v, list) else v for k, v in cfg.items()}
    cin, cout = cfg.pop("in_channels"), cfg.pop("out_channels")
    return DDPMB200(64, cin, cout, use_spatial_transformer=True, **cfg)


def _fcnn():
    return registry.build_module("fcnn", config=dict(input_dim=10, output_dim=1))


MODELS = {"classifier": _classifier, "vit_encoder": _vit_encoder, "tet_encoder": _tet_encoder, "clip": _clip, "ddpm": _ddpm,
          "fcnn": _fcnn}


@pytest.mark.parametrize("name", sorted(MODELS))
def test_every_parameter_is_in_exactly_one_arena(name):
    m = MODELS[name]()
    held = [id(p) for a in m.arenas() for p in a.params.values()]
    assert len(held) == len(set(held))
    assert set(held) == {id(p) for p in m.parameters()}


@pytest.mark.parametrize("name,sites", [("classifier", 1), ("clip", 2), ("ddpm", 1)])
def test_native_reducers_sit_on_every_exchange_site_and_no_sync_lifts_them(name, sites):
    m = MODELS[name]()
    comm = _Comm()
    reds = dp.attach_native_reducers(m, comm)
    assert len(reds) == len(m.exchanges()) == sites and m.comm is comm
    for site, red in zip(m.exchanges(), reds):
        assert site.reducer is red and red.comm is comm and red.engine is site and red.arena is site.arena
        assert site.arena in m.arenas()
        spans = sorted(s for runs in red.buckets.values() for s in runs)  # the buckets tile the site's arena
        assert spans[0][0] == 0 and spans[-1][1] == site.arena.total
        assert all(hi == lo for (_, hi), (lo, _) in zip(spans, spans[1:]))
    assert dp.attach_native_reducers(m, comm) == reds  # attached already: kept
    with dp.no_sync(m):
        assert all(site.reducer is None for site in m.exchanges()) and m.comm is None
    assert [site.reducer for site in m.exchanges()] == reds and m.comm is comm
    dp.detach_reducers(m)
    assert all(site.reducer is None for site in m.exchanges()) and m.comm is None


def test_fcnn_refuses_the_bucketed_exchange_by_name():
    with pytest.raises(NotImplementedError, match="FCNNB200"):
        dp.attach_native_reducers(_fcnn(), _Comm())


def test_graphed_trainer_leaves_the_model_alone():
    m = _classifier()
    with pytest.raises(RuntimeError):  # the capture needs CUDA
        B200TrainStep(m, ArenaAdam(m, capturable=True), clip_norm=1.0, graph=True, batch=4)
    assert not hasattr(m, "clip_norm_hook")
