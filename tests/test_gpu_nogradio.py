"""-m gpu: the `editany_nogradio.py` flow on CUDA (real kernels, synthetic test-sized checkpoints on disk):
constructor -> from_pretrained x 2 pipelines + 3 ControlNets -> SAM checkpoint -> input_data.pkl -> process().
The script text is this repo's wording of the reference's 15-line entry point (tests/test_nogradio_cpu.SCRIPT)."""
import pickle

import numpy as np
import pytest
import torch
from PIL import Image

from editanything_b200.sam_spec import SAM_TINY
from tests import synth_ckpt
from tests.test_app_cpu import _inputs
from tests.test_nogradio_cpu import SCRIPT, make_model_root

pytestmark = pytest.mark.gpu


def test_entry_script_on_cuda(tmp_path, monkeypatch):
    from editanything_b200.compat.run import run_script
    from editanything_b200.segment_anything import amg
    script = str(tmp_path / "nogradio_equivalent.py")
    open(script, "w").write(SCRIPT)
    make_model_root(str(tmp_path / "hub"))
    monkeypatch.setenv("EA_MODEL_ROOT", str(tmp_path / "hub"))
    work = tmp_path / "work"
    work.mkdir()
    monkeypatch.chdir(work)
    synth_ckpt.write_sam(str(work / "models" / "sam_vit_h_4b8939.pth"), SAM_TINY)
    monkeypatch.setattr(amg.SamAutomaticMaskGenerator.__init__, "__defaults__",
                        (8, 64, -1e9, -1.0, 1.0, 0.7, 0, 0.7, 512 / 1500, 1, None, 0, "binary_mask"))
    args, kwargs = _inputs()
    args = args[:8] + (128, 256, 20) + args[11:]
    kwargs["refine_image_resolution"] = 256
    with open("input_data.pkl", "wb") as f:
        pickle.dump({"args": args, "kwargs": kwargs}, f)
    g = run_script(script)
    m = g["model"]
    assert m.pipe.engine.dev.type == "cuda" and m.sam_generator.predictor.model.image_encoder.engine is not None
    assert m.tile_pipe.engine.unet is m.pipe.engine.unet
    refined, output = g["refined"], g["output"]
    assert len(output) == 2 and len(refined) == 2
    assert all(isinstance(i, Image.Image) and i.size == (192, 128) for i in output)
    assert all(isinstance(i, Image.Image) and i.size == (384, 256) for i in refined)
    assert all(np.array(i).std() > 0 for i in output + refined)
    # a second request replays the captured graphs (same shapes)
    g0 = m.pipe.engine._graph
    again = m.process(*args, **kwargs)
    assert m.pipe.engine._graph is g0 and len(again[1]) == 2
