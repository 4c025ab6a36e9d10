"""CLIP relevancy engine façade: ``interpret()`` with the reference signature (CLIP_explainability.ipynb cell 6)
on top of ``mmx_clip_*`` (include/mmx.h).  PyTorch only owns memory and streams here."""
from __future__ import annotations

import ctypes as C
import weakref
from dataclasses import dataclass, replace
from typing import Dict, Optional, Tuple

import torch

from ._lib import lib, check, ptr, current_stream, ClipConfigC, MmxError


@dataclass(frozen=True)
class ClipConfig:
    """Constructor arguments of the reference ``CLIP`` (CLIP/clip/model.py:249-262), ViT image tower."""
    embed_dim: int = 512
    image_resolution: int = 224
    vision_layers: int = 12
    vision_width: int = 768
    vision_patch_size: int = 32
    context_length: int = 77
    vocab_size: int = 49408
    transformer_width: int = 512
    transformer_heads: int = 8
    transformer_layers: int = 12

    @property
    def vision_tokens(self) -> int:
        return (self.image_resolution // self.vision_patch_size) ** 2 + 1

    @classmethod
    def from_state_dict(cls, sd: Dict[str, torch.Tensor]) -> "ClipConfig":
        """Infers every dimension from the weights exactly like ``build_model`` (CLIP/clip/model.py:405-434)."""
        if "visual.proj" not in sd:
            raise MmxError("only ViT image towers are supported (ModifiedResNet CLIP is out of the hot-path scope)")
        vision_width = sd["visual.conv1.weight"].shape[0]
        vision_layers = len([k for k in sd if k.startswith("visual.") and k.endswith(".attn.in_proj_weight")])
        patch = sd["visual.conv1.weight"].shape[-1]
        grid = round((sd["visual.positional_embedding"].shape[0] - 1) ** 0.5)
        width = sd["ln_final.weight"].shape[0]
        layers = len(set(k.split(".")[2] for k in sd if k.startswith("transformer.resblocks")))
        return cls(sd["text_projection"].shape[1], patch * grid, vision_layers, vision_width, patch,
                   sd["positional_embedding"].shape[0], sd["token_embedding.weight"].shape[0], width, width // 64, layers)

    def to_c(self) -> ClipConfigC:
        return ClipConfigC(self.embed_dim, self.image_resolution, self.vision_layers, self.vision_width,
                           self.vision_patch_size, self.context_length, self.vocab_size, self.transformer_width,
                           self.transformer_heads, self.transformer_layers)


VIT_B32 = ClipConfig()
VIT_L14_336 = ClipConfig(768, 336, 24, 1024, 14, 77, 49408, 768, 12, 12)


class ClipEngine:
    """Device-resident CLIP relevancy engine.  Plays the role of the reference's ``model`` argument of
    ``interpret()``; build it from a reference ``state_dict`` (``ClipEngine.from_state_dict(model.state_dict())``)."""

    def __init__(self, cfg: ClipConfig, state_dict: Dict[str, torch.Tensor], max_batch: int = 64, device=None):
        if not torch.cuda.is_available():
            raise MmxError("mmx_b200 needs a CUDA (sm_90a) device; there is no CPU fallback")
        self.cfg = cfg
        self.max_batch = int(max_batch)
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self._h = C.c_void_p()
        self._lib = lib()
        with torch.cuda.device(self.device):
            ccfg = cfg.to_c()
            check(self._lib.mmx_clip_create(C.byref(ccfg), self.max_batch, C.byref(self._h)))
            for name, t in state_dict.items():
                if name in ("input_resolution", "context_length", "vocab_size") or name.endswith("attn_mask"):
                    continue   # bookkeeping entries of JIT archives (CLIP/clip/model.py:437-439)
                t = t.detach().to("cpu", torch.float32).contiguous()
                check(self._lib.mmx_clip_load_tensor(self._h, name.encode(), C.c_void_p(t.data_ptr()), t.numel()))
            check(self._lib.mmx_clip_finalize(self._h))

    @classmethod
    def from_state_dict(cls, sd, max_batch: int = 64, device=None) -> "ClipEngine":
        return cls(ClipConfig.from_state_dict(sd), sd, max_batch, device)

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None and self._h.value:
                self._lib.mmx_clip_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    def eval(self):
        return self

    def zero_grad(self):
        return None

    def set_serial(self, serial: bool):
        """Measurement aid (``mmx_clip_set_serial``): both towers on one stream, so per-launch event times do not overlap."""
        with torch.cuda.device(self.device):
            check(self._lib.mmx_clip_set_serial(self._h, 1 if serial else 0))

    def _validate(self, images: torch.Tensor, tokens: torch.Tensor):
        """The C ABI takes raw pointers and no sizes: every shape it assumes is checked here.  Token ids outside the
        vocabulary raise like the reference's ``nn.Embedding`` (IndexError there, MmxError here)."""
        c = self.cfg
        if tokens.dim() != 2 or tokens.shape[1] != c.context_length:
            raise MmxError(f"tokens must be [B, {c.context_length}] (got {tuple(tokens.shape)})")
        if tokens.shape[0] < 1:
            raise MmxError("empty batch")
        if images.dim() != 4 or tuple(images.shape[1:]) != (3, c.image_resolution, c.image_resolution):
            raise MmxError(f"images must be [n, 3, {c.image_resolution}, {c.image_resolution}] (got {tuple(images.shape)})")
        if images.shape[0] not in (1, tokens.shape[0]):
            raise MmxError("images must hold 1 (repeated, as in the notebook) or B images")
        if tokens.is_floating_point():
            raise MmxError("tokens must be an integer tensor")
        lo, hi = int(tokens.min()), int(tokens.max())
        if lo < 0 or hi >= c.vocab_size:
            raise MmxError(f"token id out of range [0, {c.vocab_size}): min {lo}, max {hi}")

    # -- device path: inputs are CUDA tensors, work is enqueued on torch's current stream
    def interpret(self, images: torch.Tensor, tokens: torch.Tensor, start_layer: int = -1, start_layer_text: int = -1,
                  validate: bool = True) -> Tuple[torch.Tensor, torch.Tensor]:
        """``validate=False`` skips the shape / token-range checks (the range check reads the tokens back: one sync)."""
        if validate:
            self._validate(images, tokens)
        B = tokens.shape[0]
        n_img = images.shape[0]
        with torch.cuda.device(self.device):
            images = images.to(self.device, torch.float32).contiguous()
            tok = tokens.to(self.device, torch.int32).contiguous()
            ctx, sv = self.cfg.context_length, self.cfg.vision_tokens
            R_text = torch.empty(B, ctx, ctx, device=self.device, dtype=torch.float32)
            R_image = torch.empty(B, sv - 1, device=self.device, dtype=torch.float32)
            check(self._lib.mmx_clip_interpret_device(self._h, ptr(images), n_img, ptr(tok), B, int(start_layer),
                                                      int(start_layer_text), ptr(R_text), ptr(R_image), current_stream()))
        return R_text, R_image

    # -- host path: numpy / CPU tensors in, CPU tensors out; copies are inside the C call
    def interpret_host(self, images: torch.Tensor, tokens: torch.Tensor, start_layer: int = -1, start_layer_text: int = -1,
                       out: Tuple[torch.Tensor, torch.Tensor] | None = None):
        if images.is_cuda or tokens.is_cuda:
            raise MmxError("interpret_host takes host tensors (use interpret for CUDA tensors)")
        self._validate(images, tokens)
        B, n_img = tokens.shape[0], images.shape[0]
        images = images.to(torch.float32).contiguous()
        tok = tokens.to(torch.int32).contiguous()
        ctx, sv = self.cfg.context_length, self.cfg.vision_tokens
        if out is None:
            out = (torch.empty(B, ctx, ctx, dtype=torch.float32).pin_memory(),
                   torch.empty(B, sv - 1, dtype=torch.float32).pin_memory())
        elif (tuple(out[0].shape) != (B, ctx, ctx) or tuple(out[1].shape) != (B, sv - 1) or out[0].dtype != torch.float32
              or out[1].dtype != torch.float32 or not out[0].is_contiguous() or not out[1].is_contiguous()):
            raise MmxError(f"out must be contiguous fp32 ([{B},{ctx},{ctx}], [{B},{sv - 1}])")
        with torch.cuda.device(self.device):
            check(self._lib.mmx_clip_interpret_host(self._h, ptr(images), n_img, ptr(tok), B, int(start_layer),
                                                    int(start_layer_text), ptr(out[0]), ptr(out[1])))
        return out

    def tap(self, what: str, tower: int = 0, layer: int = 0) -> torch.Tensor:
        """Copy of an intermediate of the last interpret call (tower 0 = vision, 1 = text):
        - of block ``layer``: 'A', 'dA' [B,H,S,S], 'Abar' [B,S,S], 'xmid' [M,D], 'qkv' [M,3D], 'f' [M,4D] (fc1 before
          the activation), 'stats' [4,M] (mean1, rstd1, mean2, rstd2); 'x' [M,D] for layer 0 .. L (the input of block
          ``layer``; layer L is the tower output);
        - of the tower (``layer`` ignored): 'feat', 'featn', 'dfeat' [B,E] (dfeat carries the factor gscale), 'gscale' [B];
        - 'logits' [B,B].
        M = B*S, except for the ragged text tower: its rows are packed, sample b's at offs[b] .. offs[b] + len[b] - 1
        (len[b] = first argmax of its tokens + 1), and M = sum(len) of the last call."""
        p = C.c_void_p()
        dims = (C.c_int * 4)()
        ld = C.c_int()
        check(self._lib.mmx_clip_tap(self._h, what.encode(), tower, layer, C.byref(p), C.byref(dims), C.byref(ld)))
        shape = [d for d in dims]
        n_lead = 1
        nd = {"A": 4, "dA": 4, "Abar": 3, "logits": 2, "x": 2, "xmid": 2, "qkv": 2, "f": 2, "stats": 2, "feat": 2, "featn": 2,
              "dfeat": 2, "gscale": 1}[what]
        shape = shape[:nd]
        for d in shape[:-1]:
            n_lead *= d
        flat = torch.empty(n_lead * ld.value, device=self.device, dtype=torch.float32)
        torch.cuda.synchronize(self.device)
        check(self._lib.mmx_memcpy_d2d(ptr(flat), p, flat.numel() * 4, current_stream()))
        torch.cuda.synchronize(self.device)
        return flat.view(n_lead, ld.value)[:, :shape[-1]].reshape(shape).clone()


# Engines built from reference ``CLIP`` modules, keyed by the module object (dropped with it).  The engine holds a COPY of
# the weights taken at the first call; ``refresh_engine(model)`` rebuilds it after the module's weights changed.
_ENGINES: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()


def engine_for(model, device=None, max_batch: int = 64) -> ClipEngine:
    """The :class:`ClipEngine` behind ``model``: the engine itself, or one built (once) from a reference
    ``CLIP`` ``nn.Module``'s ``state_dict()`` (CLIP/clip/model.py:249; ``clip.load(...)[0]`` in the notebook)."""
    if isinstance(model, ClipEngine):
        return model
    if not (hasattr(model, "state_dict") and callable(model.state_dict)):
        raise MmxError("model must be a mmx_b200.ClipEngine or a reference CLIP nn.Module (anything with state_dict())")
    eng = _ENGINES.get(model)
    if eng is None:
        dev = device
        if dev is None or (isinstance(dev, str) and dev == "cuda"):
            dev = None
        sd = model.state_dict()
        cfg = ClipConfig.from_state_dict(sd)
        try:       # a module built with explicit constructor arguments may not follow build_model's heads = width // 64
            cfg = replace(cfg, transformer_heads=int(model.transformer.resblocks[0].attn.num_heads))
        except (AttributeError, IndexError, KeyError, TypeError):
            pass
        eng = ClipEngine(cfg, sd, max_batch=max_batch, device=dev)
        _ENGINES[model] = eng
    return eng


def refresh_engine(model) -> None:
    """Forget the engine cached for a reference module (call after its weights changed)."""
    _ENGINES.pop(model, None)


def interpret(image, texts, model, device=None, start_layer=-1, start_layer_text=-1):
    """Drop-in for the notebook's ``interpret`` (CLIP_explainability.ipynb:151-208).

    ``image``: [1,3,R,R] (repeated for every text, :153) or [B,3,R,R] (one image per text); ``texts``: [B,ctx] token
    ids; ``model``: a :class:`ClipEngine` or the reference ``CLIP`` module itself (an engine is built from its
    ``state_dict()`` on first use and cached).  Returns ``(text_relevance [B,ctx,ctx], image_relevance [B,S-1])`` on
    the engine's device."""
    return engine_for(model, device).interpret(image, texts, start_layer, start_layer_text)


def interpret_example(image, text, model, device=None, index=None):
    """The older, unbatched form of CLIP/example.py:8-32: ONE image [1,3,R,R] against N texts [N,ctx]; ``index`` picks
    the text whose logit is explained (``argmax`` of ``logits_per_image`` when None, :11-12); the image tower's relevance
    is accumulated over ALL blocks (:22-30) and ``R[0,0] = 0`` (:31) - which is outside the returned ``R[0,1:]``.
    The reference plots the map and returns nothing; here ``(image_relevance [S-1], logits_per_image [1,N])`` comes back."""
    eng = engine_for(model, device)
    if image.shape[0] != 1:
        raise MmxError("example.interpret takes one image")
    # every (image, text_n) pair in one pass: pair n's objective is logits_per_image[0, n] (pairs are independent)
    _, R_image = eng.interpret(image, text, 0, eng.cfg.transformer_layers - 1)
    logits = eng.tap("logits")[:1]                                  # [1, N]: the image against every text
    n = int(logits.argmax(-1)) if index is None else int(index)
    return R_image[n], logits
