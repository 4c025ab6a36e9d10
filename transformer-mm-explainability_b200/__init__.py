"""mmx_b200 - H100-native (sm_90a) gradient-weighted attention-relevancy engine.

Host-side mirror of the reference's Python API (hila-chefer/Transformer-MM-Explainability) over the C ABI of
libmmx.so (include/mmx.h).  Names, argument meaning and error behaviour follow the reference:

  * ``interpret(image, texts, model, device, start_layer=-1, start_layer_text=-1)``  - CLIP_explainability.ipynb cell 6
  * ``show_image_relevance``, ``generate_visualization``, ``save_image_vis``, ``show_heatmap_on_text``  - the notebooks'
    visualisation step, returning device tensors (``visualize.py``)
  * ``avg_heads``, ``apply_self_attention_rules``, ``apply_mm_attention_rules``, ``handle_residual``,
    ``compute_rollout_attention``  - DETR/modules/ExplanationGenerator.py:5-53, lxmert/lxmert/src/ExplanationGenerator.py:5-54

All arithmetic runs in hand-written CUDA kernels; there is no CPU or PyTorch fallback (``MmxError`` is raised when
the library is missing or no sm_90 GPU is present).
"""
from ._lib import MmxError, lib, LIB_PATH, exported_symbols  # noqa: F401
from .rules import (avg_heads, avg_heads_batched, apply_self_attention_rules, apply_mm_attention_rules,  # noqa: F401
                    apply_mm_attention_rules_lxmert, handle_residual, compute_rollout_attention, self_update, minmax_normalize, otsu_masks)
from .clip import ClipConfig, ClipEngine, interpret, interpret_example, engine_for, refresh_engine, VIT_B32, VIT_L14_336  # noqa: F401
from .synthetic import (clip_init_state_dict, clip_synthetic_inputs, DetrConfig, DETR_R50, DETR_TINY, detr_init_state_dict,  # noqa: F401
                        detr_sine_position_embedding, detr_synthetic_inputs, LxmertConfig, LXMERT_BASE, LXMERT_TINY,
                        lxmert_init_state_dict, lxmert_synthetic_inputs)
from .vit import ViTEngine, generate_relevance  # noqa: F401
from .detr import (DetrEngine, Generator, GeneratorAlbationNoAgg, MaskGenerator, PostProcess, PostProcessSegm,  # noqa: F401
                   detr_postprocess)
from .backbone import DetrBackbone  # noqa: F401
from .criterion import HungarianMatcher, SetCriterion  # noqa: F401
from .lxmert import LxmertEngine, GeneratorOurs, GeneratorBaselines, GeneratorOursAblationNoAggregation  # noqa: F401
from .visualbert import VisualBertEngine, SelfAttentionGenerator  # noqa: F401
from .visualize import show_image_relevance, generate_visualization, save_image_vis, show_heatmap_on_text  # noqa: F401
from .perturbation import LxmertPerturbation, VisualBertPerturbation, PERT_STEPS, topk_select  # noqa: F401

__all__ = ["MmxError", "lib", "interpret", "ClipEngine", "ClipConfig", "avg_heads", "avg_heads_batched",
           "apply_self_attention_rules", "apply_mm_attention_rules", "apply_mm_attention_rules_lxmert",
           "handle_residual", "compute_rollout_attention", "self_update", "VIT_B32", "VIT_L14_336"]
