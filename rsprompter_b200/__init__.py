"""rsprompter_b200 -- H100-native (sm_90a) implementation of the RSPrompter inference hot path.

Importing the package registers the reference's model names (``RSSamVisionEncoder``,
``RSPrompterAnchor`` ...) in the mmengine-style ``MODELS`` registry, the same effect as the
reference's ``custom_imports=['mmdet.rsprompter']`` (configs/rsprompter/_base_/rsprompter_anchor.py:3).
The CUDA extension (``librsp_b200.so``) is mandatory: there is no CPU or eager fallback.
"""
from . import _lib  # noqa: F401  (fails loudly when the extension is missing)
from .registry import MODELS, BaseModule, Config, ConfigDict, DetDataSample, InstanceData, PixelData  # noqa: F401
from . import sam_encoder  # noqa: F401

__version__ = "0.1.0"
from . import sam_decoder  # noqa: F401,E402
from . import necks, anchor_heads, query_heads, preprocess, detectors, sam_model  # noqa: F401,E402
