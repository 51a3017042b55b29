"""mmengine-compatible registry / config surface for the RSPrompter hot path.

The reference exposes its models through ``mmdet.registry.MODELS`` (mmdet/registry.py:61) and
python config files resolved by ``mmengine.Config.fromfile`` (``_base_`` inheritance,
``_delete_`` keys, ``custom_imports``; configs/rsprompter/_base_/rsprompter_anchor.py:1-3).
When mmengine/mmdet are importable the real registry is used and our classes are registered
into it (``force=True``) so ``MODELS.build(cfg.model)`` returns the H100 implementation.
This container (and the GPU box) has neither, so a minimal work-alike is provided: same
decorator, same ``build(dict(type=...))`` contract, same config-file semantics, same
``InstanceData`` / ``DetDataSample`` attribute containers the predict() methods fill in.
"""
from __future__ import annotations

import copy
import importlib
import os.path as osp
from typing import Any, Callable

import torch
from torch import nn

try:  # pragma: no cover - not available in this image
    from mmengine.config import Config, ConfigDict  # type: ignore
    from mmengine.model import BaseModule  # type: ignore
    from mmengine.structures import InstanceData, PixelData  # type: ignore
    from mmdet.registry import MODELS as _MMDET_MODELS  # type: ignore
    from mmdet.structures import DetDataSample  # type: ignore
    HAVE_MMENGINE = True
except Exception:  # noqa: BLE001
    HAVE_MMENGINE = False

# Stock mmdet component names this package also implements (inference-only, for the RSPrompter configs).  Inside a real
# mmdet process they must not displace the upstream classes other detectors rely on (samdet's FasterRCNN, samseg-*):
# they are registered only when the name is still free; the RSPrompter-specific names are re-registered with force=True.
_GENERIC_NAMES = frozenset({"RPNHead", "Shared2FCBBoxHead", "SingleRoIExtractor", "RoIAlign", "DetDataPreprocessor",
                            "AnchorGenerator", "DeltaXYWHBBoxCoder", "MSDeformAttnPixelDecoder", "StandardRoIHead",
                            "FCNMaskHead", "Mask2FormerHead", "MaskFormerFusionHead"})

if HAVE_MMENGINE:  # pragma: no cover - not available in this image

    class _ScopedModels:
        """mmdet.registry.MODELS with the registration policy above; everything else is forwarded."""

        def __init__(self, reg):
            self._reg = reg

        def register_module(self, name=None, force=False, module=None):
            def _register(cls):
                key = name or cls.__name__
                if key in _GENERIC_NAMES and self._reg.get(key) is not None:
                    return cls                      # upstream class stays
                self._reg.register_module(name=name, force=force, module=cls)
                return cls
            return _register(module) if module is not None else _register

        def __getattr__(self, item):
            return getattr(self._reg, item)

        def __contains__(self, key):
            return key in self._reg

    MODELS = _ScopedModels(_MMDET_MODELS)


if not HAVE_MMENGINE:

    class ConfigDict(dict):
        """dict with attribute access (mmengine.ConfigDict work-alike)."""

        def __getattr__(self, name: str) -> Any:
            try:
                return self[name]
            except KeyError as e:
                raise AttributeError(name) from e

        def __setattr__(self, name: str, value: Any) -> None:
            self[name] = value

        def __deepcopy__(self, memo):
            return ConfigDict({k: copy.deepcopy(v, memo) for k, v in self.items()})

    def _to_cfg(obj: Any) -> Any:
        if isinstance(obj, dict):
            return ConfigDict({k: _to_cfg(v) for k, v in obj.items()})
        if isinstance(obj, list):
            return [_to_cfg(v) for v in obj]
        if isinstance(obj, tuple):
            return tuple(_to_cfg(v) for v in obj)
        return obj

    def _merge(base: dict, child: dict) -> dict:
        """mmengine Config._merge_a_into_b: child overrides base, ``_delete_`` replaces."""
        out = dict(base)
        for k, v in child.items():
            if isinstance(v, dict):
                v = dict(v)
                delete = v.pop("_delete_", False)
                if k in out and isinstance(out[k], dict) and not delete:
                    out[k] = _merge(out[k], v)
                else:
                    out[k] = _merge({}, v)
            else:
                out[k] = v
        return out

    class Config:
        """Subset of mmengine.Config: python config files with ``_base_`` / ``_delete_``."""

        def __init__(self, cfg_dict: dict | None = None, filename: str | None = None):
            object.__setattr__(self, "_cfg_dict", _to_cfg(cfg_dict or {}))
            object.__setattr__(self, "filename", filename)

        @staticmethod
        def _file2dict(filename: str) -> dict:
            filename = osp.abspath(osp.expanduser(filename))
            if not osp.isfile(filename):
                raise FileNotFoundError(filename)
            with open(filename, encoding="utf-8") as f:
                src = f.read()
            ns: dict = {"__file__": filename}
            exec(compile(src, filename, "exec"), ns)  # noqa: S102 - config files are python
            cfg = {k: v for k, v in ns.items()
                   if not k.startswith("__") and not callable(v) and not isinstance(v, type(osp))}
            base = cfg.pop("_base_", None)
            if base is not None:
                bases = [base] if isinstance(base, str) else list(base)
                merged: dict = {}
                for b in bases:
                    bd = Config._file2dict(osp.join(osp.dirname(filename), b))
                    dup = set(merged) & set(bd)
                    if dup:
                        raise KeyError(f"duplicate keys between bases: {sorted(dup)}")
                    merged.update(bd)
                cfg = _merge(merged, cfg)
            return cfg

        @staticmethod
        def fromfile(filename: str, import_custom_modules: bool = True) -> "Config":
            cfg = Config(Config._file2dict(filename), filename=filename)
            ci = cfg.get("custom_imports")
            if import_custom_modules and ci:
                for mod in ci.get("imports", []):
                    # configs say 'mmdet.rsprompter'; this package provides those classes
                    target = "rsprompter_b200" if mod == "mmdet.rsprompter" else mod
                    try:
                        importlib.import_module(target)
                    except ImportError:
                        if not ci.get("allow_failed_imports", False):
                            raise
            return cfg

        def merge_from_dict(self, options: dict) -> None:
            """``--cfg-options`` style dotted-key overrides."""
            cfg = self._cfg_dict
            for key, val in options.items():
                d = cfg
                parts = key.split(".")
                for p in parts[:-1]:
                    d = d.setdefault(p, ConfigDict())
                d[parts[-1]] = _to_cfg(val)

        def get(self, key: str, default: Any = None) -> Any:
            return self._cfg_dict.get(key, default)

        def __getattr__(self, name: str) -> Any:
            return getattr(self._cfg_dict, name)

        def __getitem__(self, name: str) -> Any:
            return self._cfg_dict[name]

        def __contains__(self, name: str) -> bool:
            return name in self._cfg_dict

        def to_dict(self) -> dict:
            return copy.deepcopy(dict(self._cfg_dict))

    class Registry:
        """``register_module`` / ``build`` with the mmengine calling conventions."""

        def __init__(self, name: str):
            self.name = name
            self._modules: dict[str, type] = {}

        def register_module(self, name: str | None = None, force: bool = False,
                            module: type | None = None) -> Callable | type:
            def _register(cls: type) -> type:
                key = name or cls.__name__
                if key in self._modules and not force and self._modules[key] is not cls:
                    raise KeyError(f"{key} is already registered in {self.name}")
                self._modules[key] = cls
                return cls

            if module is not None:
                return _register(module)
            return _register

        def get(self, key: str) -> type | None:
            if key in self._modules:
                return self._modules[key]
            # scoped names: 'mmdet.RPNHead', 'mmpretrain.ViTSAM'
            if "." in key:
                return self._modules.get(key.split(".", 1)[1])
            return None

        def __contains__(self, key: str) -> bool:
            return self.get(key) is not None

        def build(self, cfg: dict, *args: Any, **kwargs: Any) -> Any:
            if cfg is None:
                return None
            if not isinstance(cfg, dict) or "type" not in cfg:
                raise TypeError(f"cfg must be a dict with a 'type' key, got {cfg!r}")
            cfg = dict(cfg)
            typ = cfg.pop("type")
            cls = typ if isinstance(typ, type) else self.get(typ)
            if cls is None:
                raise KeyError(f"{typ} is not in the {self.name} registry")
            for k, v in kwargs.items():
                cfg.setdefault(k, v)
            return cls(*args, **cfg)

    MODELS = Registry("model")

    class BaseModule(nn.Module):
        """mmengine.model.BaseModule work-alike: ``init_cfg`` + ``init_weights``."""

        def __init__(self, init_cfg: dict | None = None):
            super().__init__()
            self.init_cfg = copy.deepcopy(init_cfg)
            self._is_init = False

        def init_weights(self) -> None:
            for m in self.children():
                if hasattr(m, "init_weights"):
                    m.init_weights()
            self._is_init = True

    class InstanceData:
        """Per-image result container (mmengine.structures.InstanceData work-alike):
        attribute fields of equal length, ``len()`` and tensor / slice indexing."""

        def __init__(self, metainfo: dict | None = None, **fields: Any):
            object.__setattr__(self, "_fields", {})
            object.__setattr__(self, "_metainfo", dict(metainfo or {}))
            for k, v in fields.items():
                setattr(self, k, v)

        def __setattr__(self, name: str, value: Any) -> None:
            self._fields[name] = value

        def __getattr__(self, name: str) -> Any:
            fields = object.__getattribute__(self, "_fields")
            if name in fields:
                return fields[name]
            meta = object.__getattribute__(self, "_metainfo")
            if name in meta:
                return meta[name]
            raise AttributeError(name)

        def __delattr__(self, name: str) -> None:
            del self._fields[name]

        def __contains__(self, name: str) -> bool:
            return name in self._fields

        def get(self, name: str, default: Any = None) -> Any:
            return self._fields.get(name, default)

        def pop(self, name: str, *default: Any) -> Any:
            return self._fields.pop(name, *default)

        def keys(self):
            return self._fields.keys()

        def __len__(self) -> int:
            for v in self._fields.values():
                return len(v)
            return 0

        def __getitem__(self, item: Any) -> "InstanceData":
            out = InstanceData(metainfo=self._metainfo)
            for k, v in self._fields.items():
                out._fields[k] = v[item]
            return out

        def to(self, *args: Any, **kwargs: Any) -> "InstanceData":
            out = InstanceData(metainfo=self._metainfo)
            for k, v in self._fields.items():
                out._fields[k] = v.to(*args, **kwargs) if hasattr(v, "to") else v
            return out

        def cpu(self) -> "InstanceData":
            return self.to("cpu")

    class PixelData:
        """Per-image pixel-map container (mmengine.structures.PixelData work-alike): attribute fields holding
        [C, H, W] tensors (``pred_panoptic_seg.sem_seg``), ``.to`` / ``.cpu``."""

        def __init__(self, metainfo: dict | None = None, **fields: Any):
            object.__setattr__(self, "_fields", {})
            object.__setattr__(self, "_metainfo", dict(metainfo or {}))
            for k, v in fields.items():
                setattr(self, k, v)

        def __setattr__(self, name: str, value: Any) -> None:
            self._fields[name] = value

        def __getattr__(self, name: str) -> Any:
            fields = object.__getattribute__(self, "_fields")
            if name in fields:
                return fields[name]
            meta = object.__getattribute__(self, "_metainfo")
            if name in meta:
                return meta[name]
            raise AttributeError(name)

        def __contains__(self, name: str) -> bool:
            return name in self._fields

        def get(self, name: str, default: Any = None) -> Any:
            return self._fields.get(name, default)

        def keys(self):
            return self._fields.keys()

        def to(self, *args: Any, **kwargs: Any) -> "PixelData":
            out = PixelData(metainfo=self._metainfo)
            for k, v in self._fields.items():
                out._fields[k] = v.to(*args, **kwargs) if hasattr(v, "to") else v
            return out

        def cpu(self) -> "PixelData":
            return self.to("cpu")

    class DetDataSample:
        """mmdet.structures.DetDataSample work-alike: metainfo + prediction slots."""

        def __init__(self, metainfo: dict | None = None):
            self._metainfo = dict(metainfo or {})
            self._data: dict[str, Any] = {}

        @property
        def metainfo(self) -> dict:
            return self._metainfo

        def set_metainfo(self, meta: dict) -> None:
            self._metainfo.update(meta)

        def get(self, name: str, default: Any = None) -> Any:
            if name in self._data:
                return self._data[name]
            return self._metainfo.get(name, default)

        def __getattr__(self, name: str) -> Any:
            if name.startswith("_"):
                raise AttributeError(name)
            data = self.__dict__.get("_data", {})
            if name in data:
                return data[name]
            meta = self.__dict__.get("_metainfo", {})
            if name in meta:
                return meta[name]
            raise AttributeError(name)

        def __setattr__(self, name: str, value: Any) -> None:
            if name.startswith("_"):
                object.__setattr__(self, name, value)
            else:
                self._data[name] = value

        def __contains__(self, name: str) -> bool:
            return name in self._data


def make_data_samples(batch: int, size: int | tuple[int, int]) -> list:
    """Metainfo the predict() methods read (M:649-651,681-685,1754-1776) for synthetic inputs."""
    hw = (size, size) if isinstance(size, int) else tuple(size)
    return [DetDataSample(metainfo=dict(img_shape=hw, ori_shape=hw, batch_input_shape=hw,
                                        pad_shape=hw, scale_factor=(1.0, 1.0)))
            for _ in range(batch)]


__all__ = ["MODELS", "Config", "ConfigDict", "BaseModule", "InstanceData", "PixelData", "DetDataSample",
           "HAVE_MMENGINE", "make_data_samples"]
