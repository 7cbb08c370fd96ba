"""LoRA merging (editanything_b200.lora, editany_lora.py:197-329) without a GPU:
  * the merged UNet and text-encoder weights equal, bit for bit, what the reference's own `load_lora_weights` makes
    on the same files (fingerprints in tests/golden/lora_reference.pt, written by oracle/make_golden_lora.py);
  * kohya layer names resolve on the diffusers key tree of full-size SD1.5 / SD2.1 UNets; bad files raise the
    reference's exceptions and change nothing;
  * the pipeline, the tile-pass sharing, EditAnythingLoraModel, the post-hoc `load_lora_weights` and an
    `editany_beauty.py`-style entry script carry the LoRA through, with the operators on the CPU emulation;
  * the engine of a merged network issues exactly the operator calls of the base one."""
import os
import pickle

import numpy as np
import pytest
import torch
from PIL import Image

from editanything_b200 import _backend
from editanything_b200 import lora as L
from editanything_b200 import weights as W
from editanything_b200.sam_spec import SAM_TINY
from editanything_b200.unet_spec import SD15, SD21, TINY, TINY21
from editanything_b200.vae_spec import VaeConfig
from tests import cpu_ops, synth_ckpt
from tests import synth_lora as SL

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lora_reference.pt")
VCFG = VaeConfig(ch=64, ch_mult=(1, 1, 1, 1), num_res_blocks=1)
BASE = "runwayml/stable-diffusion-v1-5"


@pytest.fixture
def cpu_backend():
    _backend.OPS = cpu_ops
    yield
    _backend.OPS = None


def _te_shapes(te):
    return {k: v.shape for k, v in te.state_dict().items()}


def _write_base(root, cfg=TINY):
    synth_ckpt.write_pipeline(root, cfg, VCFG, seed=SL.UNET_SEED)
    return SL.text_encoder_fp16(root)


def _lora_file(path, cfg, te, which="both", rank=8, alpha=4.0, seed=11, dyadic=True):
    return SL.save(SL.lora_tensors(SL.case_targets(cfg, which, _te_shapes(te)), rank, alpha, seed, dyadic), path)


# ----------------------------------------------------------------------------------------------- golden
@pytest.mark.parametrize("name", list(SL.CASES))
def test_merge_matches_reference_golden(name, tmp_path, cpu_backend):
    from editanything_b200.loading import load_pipeline_parts
    want = torch.load(GOLDEN)[name]
    cfg = SL.CASES[name][0]
    root = str(tmp_path / "base")
    te_base = _write_base(root, cfg)
    paths, mult, _ = SL.write_case(name, str(tmp_path / "lora"), _te_shapes(te_base))
    ucfg, usd, _, te, _, _ = load_pipeline_parts(root, torch.device("cpu"), lora=[(p, mult) for p in paths])
    base = SL.unet_diffusers_state_dict(cfg)
    km = W.key_map(ucfg, "unet", usd.keys())
    assert ucfg == cfg and (want["unet"] or want["text_encoder"])
    for lk, v in usd.items():
        dk = km[lk]
        if dk in want["unet"]:
            assert SL.fingerprint(v) == want["unet"][dk], dk
        elif v.dtype == torch.float16:            # merged, but the delta rounded away
            assert torch.equal(v, base[dk].half()), dk
        else:                                     # not a target: today's loading path, untouched
            assert torch.equal(v, base[dk]), dk
    before = te_base.state_dict()
    for k, v in te.state_dict().items():
        if k in want["text_encoder"]:
            assert SL.fingerprint(v) == want["text_encoder"][k], k
        else:
            assert torch.equal(v, before[k]), k


def _reenact(base16, up, down, alpha, multiplier):
    """The reference's arithmetic (editany_lora.py:241-264) on one fp16 weight."""
    up, down = up.to(torch.float32), down.to(torch.float32)
    scale = alpha / up.shape[1] if alpha else 1.0
    w = base16.clone()
    if up.dim() == 4:
        w += (multiplier * scale * torch.mm(up.squeeze(3).squeeze(2), down.squeeze(3).squeeze(2))).unsqueeze(2).unsqueeze(3)
    else:
        w += multiplier * scale * torch.mm(up, down)
    return w


@pytest.mark.parametrize("cfg", [TINY, TINY21], ids=["tiny", "tiny21"])
def test_random_values_match_reenactment(cfg, tmp_path):
    te = _write_base(str(tmp_path / "base"), cfg)
    te_before = {k: v.clone() for k, v in te.state_dict().items()}
    path = _lora_file(str(tmp_path / "r.safetensors"), cfg, te, rank=6, alpha=3.0, seed=5, dyadic=False)
    usd = SL.unet_diffusers_state_dict(cfg)
    base = dict(usd)
    L.merge([(path, 0.7)], unet_sd=usd, text_encoder=te)
    lora = L.read_lora(path)
    n = 0
    for layer, e in lora.items():
        target, _ = L.layer_tokens(layer)
        path_ = layer[len("lora_unet_" if target == "unet" else "lora_te_"):]
        if target == "unet":
            key = next(k for k in usd if k.replace(".", "_") == path_ + "_weight")
            got, base16 = usd[key], base[key].half()
        else:
            key = next(k for k in te_before if k.replace(".", "_") == path_ + "_weight")
            got, base16 = te.state_dict()[key], te_before[key]
        want = _reenact(base16, e["lora_up.weight"], e["lora_down.weight"], float(e["alpha"]), 0.7)
        assert got.dtype == torch.float16 and torch.equal(got, want), key
        assert not torch.equal(got, base16), key
        n += 1
    assert n == len(SL.unet_targets(base)) + len(SL.te_targets(te_before))


# ----------------------------------------------------------------------------------------------- names
@pytest.mark.parametrize("cfg", [SD15, SD21], ids=["sd15", "sd21"])
def test_every_kohya_name_resolves_on_full_size_unets(cfg):
    shapes = SL.unet_diffusers_shapes(cfg)          # names and shapes only: nothing is allocated
    tree = L.KeyTree(shapes)
    modules = [k[:-len(".weight")] for k in shapes if k.endswith(".weight")]
    assert len(modules) > 300
    for m in modules:
        target, tokens = L.layer_tokens(SL.kohya_name(m, "unet"))
        assert target == "unet" and L.walk(tokens, "", tree.child) == m
    # the LoRA-able layers of SD1.x are 1x1 convs for proj_in/proj_out, Linear on SD2.x
    proj = [m for m in SL.unet_targets(shapes) if m.endswith("proj_in")]
    assert proj and all(len(shapes[m + ".weight"]) == (2 if cfg.use_linear_in_transformer else 4) for m in proj)


def test_text_encoder_names_resolve(tmp_path):
    te = _write_base(str(tmp_path / "base"))
    for m in SL.te_targets(_te_shapes(te)):
        target, tokens = L.layer_tokens(SL.kohya_name(m, "te"))
        assert target == "text_encoder" and L.walk(tokens, te, L._module_child) is te.get_submodule(m)


def _bad_files(tmp_path, te):
    """(exception, file) pairs: each file has valid entries first and then one bad entry."""
    good = SL.lora_tensors(SL.case_targets(TINY, "both", _te_shapes(te)), 4, 4.0, 3)
    unknown = dict(good, **{"lora_unet_down_blocks_0_nothing_here.lora_up.weight": torch.ones(8, 4),
                            "lora_unet_down_blocks_0_nothing_here.lora_down.weight": torch.ones(4, 8),
                            "lora_unet_down_blocks_0_nothing_here.alpha": torch.tensor(4.0)})
    no_alpha = dict(good)
    no_alpha.pop(next(k for k in reversed(list(good)) if k.endswith(".alpha")))
    conv = "lora_unet_down_blocks_0_resnets_0_conv1"
    c = TINY.model_channels
    locon = dict(good, **{conv + ".lora_up.weight": torch.ones(c, 4, 1, 1), conv + ".lora_down.weight": torch.ones(4, c, 3, 3),
                          conv + ".alpha": torch.tensor(4.0)})
    return [(IndexError, SL.save(unknown, str(tmp_path / "unknown.safetensors"))),
            (KeyError, SL.save(no_alpha, str(tmp_path / "no_alpha.safetensors"))),
            (RuntimeError, SL.save(locon, str(tmp_path / "locon.safetensors")))]


def test_nothing_is_read_without_a_target():
    # a pipeline sharing an already merged UNet and text encoder: the files are not opened
    assert L.plan([("/nonexistent/lora.safetensors", 1.0)]) == []


def test_bad_files_raise_and_change_nothing(tmp_path):
    te = _write_base(str(tmp_path / "base"))
    te_before = {k: v.clone() for k, v in te.state_dict().items()}
    good = _lora_file(str(tmp_path / "good.safetensors"), TINY, te)
    usd = SL.unet_diffusers_state_dict(TINY)
    base = dict(usd)
    for exc, path in _bad_files(tmp_path, te):
        with pytest.raises(exc):
            L.merge([(good, 1.0), (path, 1.0)], unet_sd=usd, text_encoder=te)
        assert all(usd[k] is base[k] for k in base)
        assert all(torch.equal(v, te_before[k]) for k, v in te.state_dict().items())


# ----------------------------------------------------------------------------------------------- pipeline
def _model_root(root, lora_seed=11):
    """A base model, the three ControlNets EditAnythingLoraModel loads and two LoRA files (a, b)."""
    from tests.test_nogradio_cpu import make_model_root
    usd, _, cns = make_model_root(root)
    te = SL.text_encoder_fp16(os.path.join(root, *BASE.split("/")))
    a = _lora_file(os.path.join(root, "lora", "a.safetensors"), TINY, te, seed=lora_seed)
    b = _lora_file(os.path.join(root, "lora", "b.safetensors"), TINY, te, which="unet", rank=2, alpha=0.0,
                   seed=lora_seed + 1)
    return usd, cns, a, b


def _merged_ldm(lora):
    sd = SL.unet_diffusers_state_dict(TINY)
    L.merge(lora, unet_sd=sd)
    return W.diffusers_to_ldm(sd, "unet", TINY)


def _assert_same_packed(x, y):
    assert x.w.keys() == y.w.keys()
    for k in x.w:
        assert torch.equal(x.w[k], y.w[k]), k


def _assert_same_te(x, y):
    sx, sy = x.state_dict(), y.state_dict()
    assert all(torch.equal(sx[k], sy[k]) for k in sx)


def test_from_pretrained_packs_the_merged_weights_and_shares_by_lora_list(tmp_path, monkeypatch, cpu_backend):
    from editanything_b200.loading import ControlNetModel, ControlNetModel2
    from editanything_b200.nets import PackedNet
    from editanything_b200.pipeline import StableDiffusionControlNetInpaintPipeline as Pipe
    root = str(tmp_path)
    usd, cns, a, b = _model_root(root)
    monkeypatch.setenv("EA_MODEL_ROOT", root)
    cn = [ControlNetModel2.from_pretrained("shgao/edit-anything-v0-4-sd15"),
          ControlNetModel.from_pretrained("lllyasviel/control_v11p_sd15_inpaint")]
    plain = Pipe.from_pretrained(BASE, controlnet=cn)
    pipe = Pipe.from_pretrained(BASE, controlnet=cn, lora=[(a, 0.5)])
    assert plain.lora == [] and pipe.lora == [(os.path.realpath(a), 0.5)]
    dev = pipe.engine.dev
    _assert_same_packed(pipe.engine.unet, PackedNet(TINY, "unet", _merged_ldm([(a, 0.5)]), dev))
    changed = [k for k in pipe.engine.unet.w if not torch.equal(pipe.engine.unet.w[k], plain.engine.unet.w[k])]
    assert any(".qkv1." in k for k in changed) and any("proj_in" in k for k in changed)
    # the ControlNets are never touched (the reference walks pipe.unet and pipe.text_encoder only)
    for i, name in enumerate(("shgao/edit-anything-v0-4-sd15", "lllyasviel/control_v11p_sd15_inpaint")):
        _assert_same_packed(pipe.engine.cns[i], PackedNet(TINY, "controlnet", cns[name], dev))
    te = SL.text_encoder_fp16(os.path.join(root, *BASE.split("/")))
    L.merge([(a, 0.5)], text_encoder=te)
    _assert_same_te(pipe.text_encoder, te)
    # the tile pipeline shares the UNet and text encoder only under an equal LoRA list; the VAE always
    tile_cn = ControlNetModel2.from_pretrained("lllyasviel/control_v11f1e_sd15_tile")
    same = Pipe.from_pretrained(BASE, controlnet=tile_cn, share_with=pipe, lora=[(a, 0.5)])
    assert same.engine.unet is pipe.engine.unet and same.text_encoder is pipe.text_encoder and same.vae is pipe.vae
    for other in ([(a, 1.0)], [(a, 0.5), (b, 0.5)], None):
        t = Pipe.from_pretrained(BASE, controlnet=tile_cn, share_with=pipe, lora=other)
        assert t.engine.unet is not pipe.engine.unet and t.text_encoder is not pipe.text_encoder and t.vae is pipe.vae
        _assert_same_packed(t.engine.unet, PackedNet(TINY, "unet", _merged_ldm(L.normalize(other)), dev))
    _assert_same_te(pipe.text_encoder, te)                    # a second load did not merge into the shared one


def test_load_lora_weights_after_loading_equals_from_pretrained(tmp_path, monkeypatch, cpu_backend):
    from editanything_b200.app import load_lora_weights
    from editanything_b200.loading import ControlNetModel2
    from editanything_b200.pipeline import StableDiffusionControlNetInpaintPipeline as Pipe
    root = str(tmp_path)
    _, _, a, b = _model_root(root)
    monkeypatch.setenv("EA_MODEL_ROOT", root)
    cn = ControlNetModel2.from_pretrained("shgao/edit-anything-v0-4-sd15")
    tile_cn = ControlNetModel2.from_pretrained("lllyasviel/control_v11f1e_sd15_tile")
    pipe = Pipe.from_pretrained(BASE, controlnet=[cn], lora=[(a, 0.5)])
    tile = Pipe.from_pretrained(BASE, controlnet=tile_cn, share_with=pipe, lora=[(a, 0.5)])
    te_shared = {k: v.clone() for k, v in pipe.text_encoder.state_dict().items()}
    cns = list(pipe.engine.cns)
    assert load_lora_weights(pipe, b, 0.5, "cpu", torch.float32) is pipe
    want = Pipe.from_pretrained(BASE, controlnet=[cn], lora=[(a, 0.5), (b, 0.5)])
    assert pipe.lora == want.lora
    _assert_same_packed(pipe.engine.unet, want.engine.unet)
    _assert_same_te(pipe.text_encoder, want.text_encoder)
    assert pipe.engine.cns == cns                               # the packed ControlNets are kept
    assert pipe.engine.ops is cpu_ops and pipe.engine.unet.ops is cpu_ops
    # the tile pipeline that shared the UNet and text encoder is unchanged: the merge went into a copy
    assert tile.engine.unet is not pipe.engine.unet and tile.text_encoder is not pipe.text_encoder
    assert all(torch.equal(v, te_shared[k]) for k, v in tile.text_encoder.state_dict().items())
    assert not pipe.text_encoder_shared and tile.text_encoder_shared
    # a list of files, on a pipeline without LoRA whose text encoder nobody shares: merged in place
    plain = Pipe.from_pretrained(BASE, controlnet=[cn])
    te = plain.text_encoder
    assert not plain.text_encoder_shared
    load_lora_weights(plain, [a, b], 0.5, "cpu", torch.float32)
    _assert_same_packed(plain.engine.unet, want.engine.unet)
    assert plain.text_encoder is te
    _assert_same_te(te, want.text_encoder)
    # a bad file changes nothing
    engine, te_before = plain.engine, {k: v.clone() for k, v in te.state_dict().items()}
    with pytest.raises(IndexError):
        load_lora_weights(plain, _bad_files(tmp_path, te)[0][1], 1.0, "cpu", torch.float32)
    assert plain.engine is engine and plain.text_encoder is te and len(plain.lora) == 2
    assert all(torch.equal(v, te_before[k]) for k, v in te.state_dict().items())


def test_app_with_lora_runs_and_rebuilds_at_weight_one(tmp_path, monkeypatch, cpu_backend):
    from editanything_b200 import app
    from tests.test_app_cpu import FakeSam, _inputs
    root = str(tmp_path / "hub")
    _, _, a, _ = _model_root(root)
    synth_ckpt.write_unet_like(os.path.join(root, "other", "controlnet"), TINY, "controlnet", 58)
    monkeypatch.setenv("EA_MODEL_ROOT", root)
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("EA_SAVE_INPUT", "0")
    model = app.EditAnythingLoraModel(base_model_path=BASE, lora_model_path=a, use_blip=False, extra_inpaint=True,
                                      lora_weight=0.5, sam_generator=FakeSam(), mask_predictor=object())
    assert model.pipe.lora == model.tile_pipe.lora == [(os.path.realpath(a), 0.5)]
    assert model.tile_pipe.engine.unet is model.pipe.engine.unet
    args, kwargs = _inputs()
    args = args[:10] + (20,) + args[11:]
    refined, output, masks, text = model.process(*args, **kwargs)
    assert len(output) == 2 and len(refined) == 2 and all(np.array(i).std() > 0 for i in output)
    # a ControlNet switch rebuilds the generation pipeline without passing lora_weight (editany_lora.py:660-666):
    # the LoRA is merged at 1.0 from then on
    kwargs = dict(kwargs, condition_model="other/controlnet", enable_tile=False)
    model.process(*args, **kwargs)
    assert model.pipe.lora == [(os.path.realpath(a), 1.0)] and model.tile_pipe.lora == [(os.path.realpath(a), 0.5)]


BEAUTY = '''import os
import pickle
from editany_lora import EditAnythingLoraModel
sd_models_path = os.environ["EA_MODEL_ROOT"]
lora_model_path = os.path.join(sd_models_path, "lora", "a.safetensors")
model = EditAnythingLoraModel(
    base_model_path=os.path.join(sd_models_path, "chilloutmix_NiPrunedFp32Fix"),
    lora_model_path=lora_model_path,
    use_blip=False,
    extra_inpaint=True,
    lora_weight=0.5,
)
with open('input_data.pkl', 'rb') as f:
    input_data = pickle.load(f)
refined, output, ref, text = model.process(*input_data['args'], **input_data['kwargs'])
'''     # this repo's wording of editany_beauty.py's model construction (its gradio front end and downloads left out)


def test_beauty_entry_script_runs(tmp_path, monkeypatch, cpu_backend):
    from editanything_b200.compat.run import run_script
    from tests.test_app_cpu import _inputs
    hub = tmp_path / "hub"
    _, _, a, _ = _model_root(str(hub))
    os.rename(str(hub / "runwayml" / "stable-diffusion-v1-5"), str(hub / "chilloutmix_NiPrunedFp32Fix"))
    monkeypatch.setenv("EA_MODEL_ROOT", str(hub))
    script = str(tmp_path / "beauty_equivalent.py")
    open(script, "w").write(BEAUTY)
    work = tmp_path / "work"
    work.mkdir()
    monkeypatch.chdir(work)
    synth_ckpt.write_sam(str(work / "models" / "sam_vit_h_4b8939.pth"), SAM_TINY)
    from editanything_b200.segment_anything import amg
    monkeypatch.setattr(amg.SamAutomaticMaskGenerator.__init__, "__defaults__",
                        (8, 64, -1e9, -1.0, 1.0, 0.7, 0, 0.7, 512 / 1500, 1, None, 0, "binary_mask"))
    args, kwargs = _inputs()
    args = args[:8] + (64, 256, 20) + args[11:]
    with open("input_data.pkl", "wb") as f:
        pickle.dump({"args": args, "kwargs": kwargs}, f)
    g = run_script(script)
    model = g["model"]
    assert model.pipe.lora == [(os.path.realpath(a), 0.5)] and model.tile_pipe.engine.unet is model.pipe.engine.unet
    assert len(g["output"]) == 2 and len(g["refined"]) == 2
    assert all(isinstance(i, Image.Image) and i.size == (64, 64) for i in g["output"])


# ----------------------------------------------------------------------------------------------- hot path
def _trace(usd):
    from editanything_b200.denoise import DenoiseEngine, ddim_schedule
    from editanything_b200.unet_spec import make_state_dict
    from oracle.inputs import make_inputs
    from tests.test_step_trace_cpu import Recorder
    csds = [make_state_dict(TINY, "controlnet", 62 + i) for i in range(2)]
    x, ctx, hints = make_inputs(TINY, 2, 8, 7, 5, n_controlnets=2)
    rec = Recorder()
    eng = DenoiseEngine(TINY, usd, csds, torch.device("cpu"), backend=rec)
    rec.lines, rec._storages, rec._alive = [], {}, []
    ts, a, ap = ddim_schedule(50)
    rec.lines.append("== prepare")
    eng.prepare(ctx, hints, [0.5, 1.0])
    rec.lines.append("== step")
    eng.begin(x[:1, :4], guidance=7.5, use_graph=False)
    eng.step(int(ts[2]), float(a[2]), float(ap[2]))
    rec.lines.append("== eps")
    eng.eps(x, int(ts[5]))
    return rec.lines, eng


def test_merged_engine_issues_the_base_engines_operator_calls(tmp_path, monkeypatch):
    for k in ("EA_LOCKSTEP", "EA_LN_FOLD", "EA_CONCURRENT", "EA_HINT_TC"):
        monkeypatch.delenv(k, raising=False)
    te = _write_base(str(tmp_path / "base"))
    path = _lora_file(str(tmp_path / "l.safetensors"), TINY, te)
    base_lines, base_eng = _trace(W.diffusers_to_ldm(SL.unet_diffusers_state_dict(TINY), "unet", TINY))
    lora_lines, lora_eng = _trace(_merged_ldm([(path, 0.5)]))
    assert len(base_lines) > 100 and lora_lines == base_lines
    assert any(not torch.equal(lora_eng.unet.w[k], base_eng.unet.w[k]) for k in base_eng.unet.w)
