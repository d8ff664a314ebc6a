"""Minimal stand-ins for diffusers' ConfigMixin / ModelMixin surface that the reference's callers touch
(train.py:86-101,230,797,851-855; models/pipeline.py:107): `.config.<key>`, `.dtype`, `.device`, `from_pretrained`
(config.json + diffusion_pytorch_model.{safetensors,bin}), `from_config`, `save_pretrained`."""
from __future__ import annotations

import inspect
import json
import os
from collections import OrderedDict

import torch
import torch.nn as nn


class FrozenConfig(OrderedDict):
    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError as e:
            raise AttributeError(name) from e


def capture_config(obj, init, args, kwargs):
    sig = inspect.signature(init)
    names = [n for n in sig.parameters if n != "self"]
    cfg = {n: sig.parameters[n].default for n in names if sig.parameters[n].kind not in
           (inspect.Parameter.VAR_KEYWORD, inspect.Parameter.VAR_POSITIONAL)}
    for n, a in zip(names, args):
        cfg[n] = a
    cfg.update({k: v for k, v in kwargs.items() if k in cfg})
    object.__setattr__(obj, "_config", FrozenConfig(cfg))


class ModelBase(nn.Module):
    config_name = "config.json"
    weights_name = "diffusion_pytorch_model"
    weights_bin_name = None            # file name of the pickle checkpoint when it is not weights_name + ".bin"

    @property
    def config(self):
        return self._config

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    # weights converted to kernel layouts are cached; any parameter move / reload invalidates the cache
    def _apply(self, fn, *a, **k):
        self.__dict__["_aab_prepared"] = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self.__dict__["_aab_prepared"] = None
        return super().load_state_dict(*a, **k)

    def invalidate_prepared(self):
        self.__dict__["_aab_prepared"] = None

    def prepare_to(self, device):
        """Move a 16-bit model that still lives on the HOST to `device` with its kernel-layout weights converted on the
        host first: every converted tensor and every parameter then reaches the GPU by a plain H2D memcpy, so no torch
        cast / permute / cat kernel runs on the device at all (the lazy path, `_prepared()` on first use, converts on
        the GPU with a few hundred small torch copy kernels).  Returns self."""
        p0 = next(self.parameters())
        if p0.is_cuda:
            raise RuntimeError("prepare_to() converts on the host: call it before moving the model to the GPU")
        if p0.dtype not in (torch.float16, torch.bfloat16):
            raise TypeError("prepare_to() needs a 16-bit model (.to(torch.float16) / .to(torch.bfloat16) first)")
        device = torch.device(device)
        prep = self._build_prepared(p0.dtype, p0.device)

        def mv(o):
            if torch.is_tensor(o):
                return o.to(device)
            if isinstance(o, dict):
                return {k: mv(v) for k, v in o.items()}
            if isinstance(o, (list, tuple)):
                return type(o)(mv(v) for v in o)
            return o
        prep.m = {k: mv(v) for k, v in prep.m.items()}
        prep.device = device
        nn.Module._apply(self, lambda t: t.to(device))             # bypass the cache invalidation of ModelBase._apply
        self.__dict__["_aab_prepared"] = prep
        return self

    @classmethod
    def from_config(cls, config, **overrides):
        sig = inspect.signature(cls.__init__).parameters
        kw = {k: v for k, v in dict(config).items() if k in sig}
        kw.update({k: v for k, v in overrides.items() if k in sig})
        return cls(**kw)

    @classmethod
    def _weight_files(cls, variant=None):
        """(safetensors name, pickle name) of the checkpoint; a `variant` goes before the extension, as diffusers and
        transformers name it (`diffusion_pytorch_model.fp16.safetensors`, `pytorch_model.fp16.bin`)."""
        names = (cls.weights_name + ".safetensors", cls.weights_bin_name or (cls.weights_name + ".bin"))
        if variant is None:
            return names
        return tuple(f"{stem}.{variant}{ext}" for stem, ext in (os.path.splitext(n) for n in names))

    @classmethod
    def from_pretrained(cls, path, subfolder=None, torch_dtype=None, ignore_mismatched_sizes=False,
                        low_cpu_mem_usage=False, device_map=None, variant=None, **overrides):
        root = os.path.join(path, subfolder) if subfolder else path
        with open(os.path.join(root, cls.config_name)) as f:
            cfg = {k: v for k, v in json.load(f).items() if not k.startswith("_")}
        st_name, bin_name = cls._weight_files(variant)
        if variant is not None and not any(os.path.exists(os.path.join(root, n)) for n in (st_name, bin_name)):
            plain = cls._weight_files()
            found = [n for n in plain if os.path.exists(os.path.join(root, n))]
            raise FileNotFoundError(f"no {st_name} or {bin_name} in {root} (variant={variant!r})"
                                    + (f"; {found[0]} exists: load it without `variant`" if found else
                                       f", and no {plain[0]} or {plain[1]} either"))
        model = cls.from_config(cfg, **overrides)
        st_path = os.path.join(root, st_name)
        if os.path.exists(st_path):
            from safetensors.torch import load_file
            sd = load_file(st_path)
        else:
            sd = torch.load(os.path.join(root, bin_name), map_location="cpu")
        if ignore_mismatched_sizes:
            own = model.state_dict()
            sd = {k: v for k, v in sd.items() if k in own and own[k].shape == v.shape}
        sd = model._convert_legacy_keys(sd)
        missing, unexpected = model.load_state_dict(sd, strict=False)
        if unexpected:
            raise ValueError(f"unexpected keys in checkpoint: {unexpected[:8]} ...")
        model._missing_keys = missing
        if torch_dtype is not None:
            model = model.to(torch_dtype)
        return model.eval()

    def _convert_legacy_keys(self, sd):
        return sd

    def save_pretrained(self, path, safe_serialization=True):
        os.makedirs(path, exist_ok=True)
        cfg = {k: (list(v) if isinstance(v, tuple) else v) for k, v in self.config.items()}
        cfg["_class_name"] = type(self).__name__
        with open(os.path.join(path, self.config_name), "w") as f:
            json.dump(cfg, f, indent=2)
        sd = {k: v.contiguous() for k, v in self.state_dict().items()}
        if safe_serialization:
            from safetensors.torch import save_file
            save_file(sd, os.path.join(path, self.weights_name + ".safetensors"))
        else:
            torch.save(sd, os.path.join(path, self.weights_name + ".bin"))


class BaseOutput(dict):
    """Tiny output record: attribute + index access like diffusers' BaseOutput."""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.__dict__.update(kw)

    def __getitem__(self, k):
        if isinstance(k, int):
            return list(self.values())[k]
        return super().__getitem__(k)
