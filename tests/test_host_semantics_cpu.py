"""Host semantics of SURVEY.md §8a rows R2 / R3 / R4 (`editanything_b200.host`) against what the REFERENCE's own
functions return on the same inputs: annotator/util.py's helpers and show_anns / make_inpaint_condition /
get_pipeline_embeds of editany_lora.py were run once by oracle/make_golden_host.py, which stored bit-exact
fingerprints (dtype, shape, sha256 of the bytes) of their results in tests/golden/host_reference.pt."""
import hashlib
import os
from types import SimpleNamespace

import numpy as np
import torch
from PIL import Image

from editanything_b200 import host

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "host_reference.pt")


def fingerprint(x):
    """Structure-preserving, bit-exact digest of what a function returned (tensors, arrays, PIL images, containers)."""
    if torch.is_tensor(x):
        a = x.detach().cpu().contiguous()
        return ("tensor", str(a.dtype), tuple(a.shape), hashlib.sha256(a.view(torch.uint8).numpy().tobytes()
                                                                       if a.numel() else b"").hexdigest())
    if isinstance(x, Image.Image):
        a = np.ascontiguousarray(np.array(x))
        return ("image", x.mode, x.size, hashlib.sha256(a.tobytes()).hexdigest())
    if isinstance(x, np.ndarray):
        a = np.ascontiguousarray(x)
        return ("ndarray", str(a.dtype), a.shape, hashlib.sha256(a.tobytes()).hexdigest())
    if isinstance(x, (list, tuple)):
        return [fingerprint(v) for v in x]
    if isinstance(x, dict):
        return {k: fingerprint(v) for k, v in x.items()}
    if isinstance(x, torch.Generator):
        return "generator"
    if isinstance(x, (np.integer, np.floating)):
        return x.item()
    return x


def golden(key):
    return torch.load(GOLD, weights_only=False)[key]


def _anns(seed, n=7, H=48, W=64):
    g = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        m = np.zeros((H, W), dtype=bool)
        y0, x0 = g.randint(0, H - 8), g.randint(0, W - 8)
        m[y0:y0 + g.randint(4, 30), x0:x0 + g.randint(4, 40)] = True
        out.append({"segmentation": m, "area": int(m.sum())})
    return out


def many_anns():
    return [{"segmentation": np.eye(300, dtype=bool)[i:i + 1].repeat(2, 0), "area": 2} for i in range(300)]


def show_anns_cases(fn):
    """show_anns on the fixed inputs, with the global numpy seed it draws its colours from."""
    np.random.seed(11)
    a = fn(_anns(3))
    np.random.seed(1)
    return {"anns3": a, "empty": fn([]), "many": fn(many_anns())[1]}


def test_show_anns_matches_reference_including_the_ordering_quirk():
    ref = golden("show_anns")
    anns = _anns(3)
    ours = show_anns_cases(host.show_anns)
    img_o, res_o = ours["anns3"]
    assert res_o.dtype == np.float64
    assert fingerprint(ours["anns3"]) == ref["anns3"]
    # the quirk: ids follow the generator's order, not the area order - sorting the input changes the map
    srt = sorted(anns, key=lambda a: a["area"], reverse=True)
    np.random.seed(11)
    assert not np.array_equal(host.show_anns(srt)[1], res_o)
    assert ours["empty"] is None and ref["empty"] is None
    # more than 255 masks: the id spills into channel 1
    assert fingerprint(ours["many"]) == ref["many"] and ours["many"][:, :, 1].max() == 1


def inpaint_condition_case(fn):
    g = np.random.RandomState(5)
    img = g.randint(0, 256, (32, 48, 3)).astype(np.uint8)
    mask = np.zeros((32, 48, 3), dtype=np.uint8)
    mask[8:20, 10:30] = 255
    return fn(img.copy(), mask)


def test_make_inpaint_condition_matches_reference():
    a = inpaint_condition_case(host.make_inpaint_condition)
    assert a.shape == (1, 3, 32, 48)
    assert fingerprint(a) == golden("make_inpaint_condition")
    assert float(a.min()) == -1.0


def image_helper_cases(U):
    """HWC3 / resize_image / resize_points / get_bounding_box of module U (host or annotator.util) on fixed inputs."""
    g = np.random.RandomState(7)
    out = {"HWC3": [U.HWC3(g.randint(0, 256, shape).astype(np.uint8))
                    for shape in [(50, 70), (50, 70, 1), (50, 70, 3), (50, 70, 4)]]}
    img = g.randint(0, 256, (300, 421, 3)).astype(np.uint8)
    out["resize_image"] = [U.resize_image(img, res) for res in (128, 512, 1024)]
    out["resize_points"] = U.resize_points([(10, 20, 1), (333, 7, 0)], img.shape, 512)
    m = np.zeros((40, 60, 3), dtype=np.uint8)
    m[5:9, 11:30] = 1
    out["get_bounding_box"] = [int(v) for v in U.get_bounding_box(m)]
    return out


def test_image_helpers_match_annotator_util():
    ours = image_helper_cases(host)
    for a in ours["resize_image"]:
        assert a.shape[0] % 64 == 0 and a.shape[1] % 64 == 0
    assert ours["get_bounding_box"] == [11, 5, 29, 8]
    assert fingerprint(ours) == golden("image_helpers")


class _Tok:
    """Word-level tokenizer with the call surface get_pipeline_embeds uses (CLIPTokenizer-like: BOS ... EOS, pad)."""
    model_max_length = 8

    def __call__(self, text, return_tensors="pt", truncation=False, padding=None, max_length=None):
        ids = [1] + [3 + (sum(map(ord, w)) % 50) for w in text.replace(",", " ").split()] + [2]
        if padding == "max_length" and max_length is not None:
            ids = ids + [0] * (max_length - len(ids))
        return SimpleNamespace(input_ids=torch.tensor([ids]))


class _Enc(torch.nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.emb = torch.nn.Embedding(64, 16)

    def forward(self, ids):
        x = self.emb(ids)
        return (x + x.cumsum(1) * 0.1,)          # depends on the position inside the window


LONG_PROMPT = "a photo of a very long prompt with many many words, best quality, extremely detailed, more words here"


def pipeline_embeds_cases(fn):
    pipe = SimpleNamespace(tokenizer=_Tok(), text_encoder=_Enc())
    return [fn(pipe, p, n, "cpu") for p, n in [(LONG_PROMPT, "lowres, bad anatomy"), ("short", LONG_PROMPT), ("a cat", "a dog")]]


def test_get_pipeline_embeds_windows_match_reference():
    ours = pipeline_embeds_cases(host.get_pipeline_embeds)
    for a in ours:
        assert a[0].shape == a[1].shape
    assert fingerprint(ours) == golden("get_pipeline_embeds")
    pipe = SimpleNamespace(tokenizer=_Tok(), text_encoder=_Enc())
    assert host.get_pipeline_embeds(pipe, LONG_PROMPT, "x", "cpu")[0].shape[1] > _Tok.model_max_length


def test_seed_everything_seeds_all_generators():
    import random
    host.seed_everything(123)
    a = (random.random(), np.random.rand(), torch.rand(1).item())
    host.seed_everything(123)
    assert a == (random.random(), np.random.rand(), torch.rand(1).item())
    assert os.environ["PL_GLOBAL_SEED"] == "123"
