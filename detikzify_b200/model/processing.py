"""
Processor (image processor + tokenizer) with the reference's call surface.

Mirrors detikzify/model/processing_detikzify.py:41-123 (prompt = image_token * image_seq_len + text,
image processor + tokenizer, ``decode`` / ``batch_decode`` passthrough) and the v1 image processor
detikzify/model/v1/processing_detikzify.py:98-124,162-253 (resize to S x S bicubic -> x 1/255 ->
(x - mean) / std with the timm SigLIP statistics 0.5 / 0.5 -> channels first).

Tokenizer files of the named checkpoints are not reachable offline, so ``SyntheticTokenizer`` is a
self-contained byte-level tokenizer with the v1 conventions (model_max_length=2048, no BOS on
encode, EOS appended on request, patch token := BOS; detikzify/model/v1/__init__.py:26-34,49).
A real HF tokenizer object can be passed instead: only the attributes used below are required.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch
from PIL import Image


class BatchFeature(dict):
    """dict with attribute access, ``.to(device)``, like HF's BatchFeature/BatchEncoding."""

    def __getattr__(self, item):
        try:
            return self[item]
        except KeyError as e:
            raise AttributeError(item) from e

    def to(self, *args, **kwargs):
        out = BatchFeature()
        for k, v in self.items():
            if isinstance(v, torch.Tensor):
                if v.is_floating_point():
                    out[k] = v.to(*args, **kwargs)
                else:  # ids keep their integer dtype (HF semantics)
                    dev = [a for a in args if isinstance(a, (str, torch.device, int))]
                    out[k] = v.to(dev[0]) if dev else (v.to(device=kwargs["device"]) if "device" in kwargs else v)
            else:
                out[k] = v
        return out


_PRECISION_BITS = 32 - 8 - 2


def _bicubic(x: float) -> float:
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


_COEFF_CACHE: Dict = {}


def pil_resample_coeffs(in_size: int, out_size: int):
    """Pillow's 8-bit bicubic resampling taps for one axis (third party: Pillow src/libImaging/Resample.c,
    ``precompute_coeffs`` + ``normalize_coeffs_8bpc``; restated, double arithmetic in the same order) ->
    (bounds int32 [out, 2] = {first input index, tap count}, coef int32 [out, ksize] 22-bit fixed point, ksize).
    The device resize (csrc/preprocess.cu) applies them exactly like Pillow does, so it is bit-identical to
    ``Image.resize(..., BICUBIC)``."""
    key = (in_size, out_size)
    if key in _COEFF_CACHE:
        return _COEFF_CACHE[key]
    import math
    support0 = 2.0
    scale = float(in_size) / out_size
    filterscale = scale if scale >= 1.0 else 1.0
    support = support0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    coef = np.zeros((out_size, ksize), dtype=np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = int(center - support + 0.5)
        if xmin < 0:
            xmin = 0
        xmax = int(center + support + 0.5)
        if xmax > in_size:
            xmax = in_size
        xmax -= xmin
        k = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        for x in range(xmax):
            v = k[x] / ww if ww != 0.0 else k[x]
            coef[xx, x] = int(-0.5 + v * (1 << _PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << _PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    out = (torch.from_numpy(bounds), torch.from_numpy(coef), ksize)
    _COEFF_CACHE[key] = out
    return out


def pil_resample_reference(arr: np.ndarray, out_size: int) -> np.ndarray:
    """numpy restatement of the two-pass fixed-point resize (what the device kernels compute): uint8 [h, w, 3] -> [S, S, 3]."""
    h, w, _ = arr.shape
    bh, ch, _ = pil_resample_coeffs(w, out_size)
    bv, cv, _ = pil_resample_coeffs(h, out_size)
    bh, ch, bv, cv = bh.numpy(), ch.numpy().astype(np.int64), bv.numpy(), cv.numpy().astype(np.int64)
    half = 1 << (_PRECISION_BITS - 1)
    tmp = np.zeros((h, out_size, 3), dtype=np.uint8)
    a64 = arr.astype(np.int64)
    for x in range(out_size):
        x0, n = bh[x]
        acc = half + (a64[:, x0:x0 + n, :] * ch[x, :n, None]).sum(axis=1)
        tmp[:, x, :] = np.clip(acc >> _PRECISION_BITS, 0, 255)
    out = np.zeros((out_size, out_size, 3), dtype=np.uint8)
    t64 = tmp.astype(np.int64)
    for y in range(out_size):
        y0, n = bv[y]
        acc = half + (t64[y0:y0 + n, :, :] * cv[y, :n, None, None]).sum(axis=0)
        out[y] = np.clip(acc >> _PRECISION_BITS, 0, 255)
    return out


class DetikzifyImageProcessor:
    model_input_names = ["pixel_values"]

    def __init__(self, size: int = 384, image_mean=(0.5, 0.5, 0.5), image_std=(0.5, 0.5, 0.5),
                 resample: int = 3, rescale_factor: float = 1 / 255):
        self.size = {"height": size, "width": size}
        self.image_mean, self.image_std = list(image_mean), list(image_std)
        self.resample, self.rescale_factor = resample, rescale_factor
        self.do_resize = self.do_rescale = self.do_normalize = True

    def to_dict(self) -> Dict:
        return dict(size=self.size, image_mean=self.image_mean, image_std=self.image_std, resample=self.resample,
                    rescale_factor=self.rescale_factor, image_size=self.size["height"],
                    image_processor_type="TimmImageProcessor")

    def preprocess(self, images, return_tensors: Optional[str] = "pt", **_) -> BatchFeature:
        if not isinstance(images, (list, tuple)):
            images = [images]
        out = []
        for im in images:
            if isinstance(im, torch.Tensor):
                im = im.numpy()
            if isinstance(im, np.ndarray):
                im = Image.fromarray(im.astype(np.uint8))
            im = im.convert("RGB")
            if im.size != (self.size["width"], self.size["height"]):
                im = im.resize((self.size["width"], self.size["height"]), resample=Image.Resampling(self.resample))
            a = np.asarray(im, dtype=np.float32) * np.float32(self.rescale_factor)
            a = (a - np.asarray(self.image_mean, dtype=np.float32)) / np.asarray(self.image_std, dtype=np.float32)
            out.append(np.ascontiguousarray(a.transpose(2, 0, 1)))
        data = np.stack(out)
        return BatchFeature(pixel_values=torch.from_numpy(data) if return_tensors == "pt" else data)

    __call__ = preprocess

    def preprocess_device(self, images, engine) -> torch.Tensor:
        """Same result as ``preprocess`` (bit-identical resize, fp32 normalisation), computed on the engine's device: the
        uint8 pixels are uploaded and resized / normalised by ``dtk_image_preprocess``. Returns ``[B, 3, S, S]`` fp32 on the
        device, ready for ``dtk_vit_encode`` — the path for bursts of candidate renders from parallel MCTS rollouts."""
        if not isinstance(images, (list, tuple)):
            images = [images]
        if self.resample != 3:
            raise ValueError("device preprocessing implements the bicubic resampler only")
        S = self.size["height"]
        out = torch.empty(len(images), 3, S, S, dtype=torch.float32, device=engine.device)
        for i, im in enumerate(images):
            if isinstance(im, torch.Tensor):
                im = im.numpy()
            if not isinstance(im, np.ndarray):
                im = np.asarray(im.convert("RGB"), dtype=np.uint8)
            arr = torch.from_numpy(np.ascontiguousarray(im.astype(np.uint8)))
            if engine.device.type == "cuda":
                arr = arr.pin_memory()
            engine.image_preprocess(arr.to(engine.device, non_blocking=True), S, self.rescale_factor, self.image_mean,
                                    self.image_std, out[i])
        return out


class SyntheticTokenizer:
    """Byte-level tokenizer over [0, vocab): ids 0..255 are bytes, a block of multi-character TikZ
    tokens follows (several contain newlines -> exercises the MCTS newline bookkeeping,
    detikzify/infer/generate.py:229-244), the rest of the id space are opaque filler tokens."""

    MULTI = ["\n\n", ";\n", "\\draw", "\\node", "\\begin{tikzpicture}", "\\end{tikzpicture}\n", " -- ", "  ",
             "\\fill", "circle", "rectangle", "[->]", "\n  ", "};\n", "cycle;\n", "\\path"]

    def __init__(self, vocab_size: int, bos_token_id: int, eos_token_id: int, pad_token_id: int,
                 model_max_length: int = 2048):
        self.vocab_size = vocab_size
        self.bos_token_id, self.eos_token_id, self.pad_token_id = bos_token_id, eos_token_id, pad_token_id
        self.bos_token, self.eos_token, self.pad_token = "<|bos|>", "<|eos|>", "<pad>"
        self.model_max_length = model_max_length
        self.padding_side = "right"
        self.init_kwargs: Dict = {}
        self.model_input_names = ["input_ids", "attention_mask"]
        self._id2tok: List[str] = []
        special = {bos_token_id: self.bos_token, eos_token_id: self.eos_token, pad_token_id: self.pad_token}
        for i in range(vocab_size):
            if i in special:
                self._id2tok.append(special[i])
            elif i < 256:
                self._id2tok.append(bytes([i]).decode("latin-1"))
            elif i - 256 < len(self.MULTI):
                self._id2tok.append(self.MULTI[i - 256])
            else:
                self._id2tok.append(f"<t{i}>")
        self.special_ids = set(special)
        self.vocab: Dict[str, int] = {t: i for i, t in enumerate(self._id2tok)}
        self._multi = sorted(((t, i) for i, t in enumerate(self._id2tok) if len(t) > 1 and i not in self.special_ids
                              and not t.startswith("<t")), key=lambda x: -len(x[0]))
        self._special_strs = [(s, i) for i, s in special.items()]

    def __len__(self):
        return self.vocab_size

    def convert_ids_to_tokens(self, ids):
        if isinstance(ids, int):
            return self._id2tok[ids]
        return [self._id2tok[i] for i in ids]

    def convert_tokens_to_ids(self, toks):
        if isinstance(toks, str):
            return self.vocab[toks]
        return [self.vocab[t] for t in toks]

    def encode(self, text: str) -> List[int]:
        ids, i = [], 0
        while i < len(text):
            for s, sid in self._special_strs:
                if text.startswith(s, i):
                    ids.append(sid)
                    i += len(s)
                    break
            else:
                for t, tid in self._multi:
                    if text.startswith(t, i):
                        ids.append(tid)
                        i += len(t)
                        break
                else:
                    for b in text[i].encode("utf-8"):
                        ids.append(b if b not in self.special_ids else ord("?"))
                    i += 1
        return ids

    def __call__(self, text=None, truncation: bool = False, max_length: Optional[int] = None,
                 return_tensors: Optional[str] = None, add_special_tokens: bool = False, padding=False, **_):
        texts = [text] if isinstance(text, str) else list(text)
        enc = [self.encode(t) for t in texts]
        if truncation:
            lim = max_length or self.model_max_length
            enc = [e[:lim] for e in enc]
        if padding and padding != "do_not_pad":   # right padding to the longest sequence
            n = max(len(e) for e in enc)
            mask = [[1] * len(e) + [0] * (n - len(e)) for e in enc]
            enc = [e + [self.pad_token_id] * (n - len(e)) for e in enc]
            if return_tensors == "pt":
                return BatchFeature(input_ids=torch.tensor(enc, dtype=torch.long), attention_mask=torch.tensor(mask, dtype=torch.long))
            return BatchFeature(input_ids=enc, attention_mask=mask)
        if return_tensors == "pt":
            n = max(len(e) for e in enc)
            if any(len(e) != n for e in enc):
                raise ValueError("ragged batch: pass one prompt at a time (the reference never batches, SURVEY B.7)")
            return BatchFeature(input_ids=torch.tensor(enc, dtype=torch.long),
                                attention_mask=torch.ones(len(enc), n, dtype=torch.long))
        return BatchFeature(input_ids=enc, attention_mask=[[1] * len(e) for e in enc])

    def decode(self, token_ids=None, skip_special_tokens: bool = False, **_) -> str:
        if isinstance(token_ids, torch.Tensor):
            token_ids = token_ids.tolist()
        if isinstance(token_ids, int):
            token_ids = [token_ids]
        parts, raw = [], bytearray()

        def flush():
            if raw:
                parts.append(raw.decode("utf-8", errors="replace"))
                raw.clear()

        for i in token_ids:
            if i in self.special_ids:
                if not skip_special_tokens:
                    flush()
                    parts.append(self._id2tok[i])
            elif i < 256:
                raw.append(i)
            else:
                flush()
                parts.append(self._id2tok[i])
        flush()
        return "".join(parts)

    def batch_decode(self, sequences, **kw) -> List[str]:
        return [self.decode(s, **kw) for s in sequences]


class DetikzifyProcessor:
    """``processor(images=, text=, return_tensors="pt", text_kwargs={...})`` ->
    {input_ids, attention_mask, pixel_values} (reference processing_detikzify.py:69-115)."""

    attributes = ["image_processor", "tokenizer"]

    def __init__(self, image_processor, tokenizer=None, image_seq_len: int = 300,
                 image_token: str = "<|reserved_special_token_2|>", model_expects_text: bool = False, **kwargs):
        if image_processor is None:
            raise ValueError("You need to specify an `image_processor`.")
        if tokenizer is None:
            raise ValueError("You need to specify a `tokenizer`.")
        if image_token not in tokenizer.vocab:
            raise ValueError(f"{image_token} needs to be added to the `tokenizer` vocabulary.")
        self.image_processor, self.tokenizer = image_processor, tokenizer
        self.image_token, self.image_seq_len = image_token, image_seq_len
        self.model_expects_text = model_expects_text

    def __call__(self, text=None, images=None, image_seq_len: Optional[int] = None, add_bos_token: bool = None,
                 add_eos_token: bool = None, return_tensors: Optional[str] = "pt", text_kwargs: Optional[dict] = None,
                 images_kwargs: Optional[dict] = None, **kwargs) -> BatchFeature:
        if images is None:
            raise ValueError("`images` are expected as arguments to a `DetikzifyProcessor` instance.")
        if isinstance(images, list) and all(isinstance(img, list) and len(img) == 1 for img in images):
            images = [img[0] for img in images]
        if not isinstance(images, (list, tuple)):
            images = [images]
        if text is None:
            text = len(images) * [""]
        elif isinstance(text, str):
            text = [text]
        if len(images) != len(text):
            raise ValueError(f"Received {len(images)} images for {len(text)} prompts. "
                             "Each prompt should be associated with an image.")
        prompts = []
        for prompt in text:
            assert self.image_token not in prompt, "Image tokens are added by the processor!"
            if add_bos_token:
                prompt += self.tokenizer.bos_token
            if add_eos_token:
                prompt += self.tokenizer.eos_token
            n = image_seq_len if image_seq_len is not None else self.image_seq_len
            prompts.append(self.image_token * n + prompt)
        tk = dict(add_special_tokens=False, padding=False)
        tk.update(text_kwargs or {})
        image_inputs = self.image_processor(images=list(images), return_tensors=return_tensors, **(images_kwargs or {}))
        text_inputs = self.tokenizer(text=prompts, return_tensors=return_tensors, **tk)
        return BatchFeature({**image_inputs, **text_inputs})

    def batch_decode(self, *args, **kwargs):
        return self.tokenizer.batch_decode(*args, **kwargs)

    def decode(self, *args, **kwargs):
        return self.tokenizer.decode(*args, **kwargs)

    @property
    def model_input_names(self):
        return list(dict.fromkeys(self.tokenizer.model_input_names + self.image_processor.model_input_names))


class AdapterProcessor:
    """TikZero processor (reference model/adapter/processing_adapter.py:20-62): the caption goes through the embedder's
    tokenizer with its keys prefixed ``adapter_``; without images the inner processor runs on ``DUMMY_IMAGE`` and only its
    ``input_ids`` / ``attention_mask`` are kept (the model feeds the adapter's learned ``dummy_input`` to the tower instead)."""

    attributes = ["processor", "tokenizer"]

    def __init__(self, processor, tokenizer=None, **kwargs):
        if processor is None:
            raise ValueError("You need to specify a `processor`.")
        if tokenizer is None:
            raise ValueError("You need to specify a `tokenizer`.")
        self.processor, self.tokenizer = processor, tokenizer

    def __call__(self, text=None, images=None, **kwargs) -> BatchFeature:
        from ..util import DUMMY_IMAGE
        if images is None and text is None:
            raise ValueError("Either `images` or `text` (or both) are expected as arguments to an `AdapterProcessor` instance.")
        text_kwargs, images_kwargs = dict(kwargs.pop("text_kwargs", None) or {}), dict(kwargs.pop("images_kwargs", None) or {})
        if text is None:
            text_inputs = dict()
        else:
            text = [text] if isinstance(text, str) else list(text)
            text_inputs = {f"adapter_{k}": v for k, v in self.tokenizer(text=text, **kwargs, **text_kwargs).items()}
            if getattr(self.processor, "model_expects_text", False):
                images_kwargs.update(text=text, add_bos_token=True)
        if images is None:
            image_inputs = self.processor(images=len(text) * [DUMMY_IMAGE], **kwargs, **images_kwargs)
            image_inputs = {k: image_inputs[k] for k in ["input_ids", "attention_mask"] if k in image_inputs}
        else:
            if not isinstance(images, (list, tuple)):
                images = [images]
            image_inputs = self.processor(images=images, **kwargs, **images_kwargs)
        if text is not None and images is not None and len(images) != len(text):
            raise ValueError(f"Received {len(images)} images for {len(text)} prompts. "
                             "Each prompt should be associated with an image.")
        return BatchFeature({**image_inputs, **text_inputs})

    def batch_decode(self, *args, **kwargs):
        return self.processor.batch_decode(*args, **kwargs)

    def decode(self, *args, **kwargs):
        return self.processor.decode(*args, **kwargs)

    @property
    def model_input_names(self):
        return list(dict.fromkeys(self.tokenizer.model_input_names + self.processor.model_input_names))
