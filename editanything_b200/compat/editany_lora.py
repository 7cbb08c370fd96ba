"""`editany_lora` as the reference's entry scripts import it (editany_nogradio.py:2, editany.py, editany_demo.py)."""
from editanything_b200.app import (EditAnythingLoraModel, config_dict, init_sam_model, load_lora_weights,  # noqa: F401
                                   obtain_generation_model, obtain_tile_model)
from editanything_b200.host import get_pipeline_embeds, make_inpaint_condition, show_anns  # noqa: F401
