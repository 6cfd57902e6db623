"""SelfSim image similarity (the MCTS reward): the model's own vision tower encodes the rendered candidate
and the input figure; mode "cos" = cosine of the attention-pooled vectors in fp64, "cos_avg" = cosine of
mean patch tokens, "emd" = 2 tanh(-EMD) + 1 of the two sets of patch tokens under the cost 1 - cos
(reference detikzify/evaluate/imagesim.py:91-125; v1 models use "cos", detikzify/model/v1/configuration_detikzify.py:11-13;
the v2 models, whose config has no pooling_mode, default to "emd": imagesim.py:64).

EMD: the reference calls POT's network simplex ``ot.lp.emd2(M=dists, a=[], b=[])`` (absent offline): both marginals are
uniform over the same number N of patches, so an optimal transport plan is a permutation (Birkhoff - von Neumann) and
EMD = min-cost perfect matching / N, solved exactly by ``scipy.optimize.linear_sum_assignment`` (Jonker-Volgenant); the test
suite checks it against the transport LP. The cost matrix (fp64 pairwise cosines) is built on the device, the N x N
assignment runs on the host like the reference's simplex (about 23 ms per pair at the v2 size N = 900).

TikZero (reference imagesim.py:61-85,87-142): with a text-conditioning adapter loaded, a side that carries a caption (the target
``img2`` or no image, plus ``text2``) is encoded by the adapted tower; the rendered candidates stay on the plain tower. The
conditioned target is encoded once per (figure, caption) and reused for every candidate.

torchmetrics is not a dependency here: the ``update / compute / reset`` protocol the MCTS driver uses
(infer/generate.py:293-298) is implemented directly.
"""
from __future__ import annotations

from typing import List, Optional, Union

import torch
import torch.nn.functional as F
from PIL import Image

from ..util.image import expand, load


class ImageSim:
    higher_is_better = True

    def __init__(self, model=None, processor=None, mode: str = "cos", preprocess: bool = True, tokenizer=None, **_):
        if mode not in ("cos", "cos_avg", "emd"):
            raise NotImplementedError(f"ImageSim mode {mode!r} is not supported (cos / cos_avg / emd)")
        self.model, self.processor = model, processor
        self.tokenizer = tokenizer          # caption tokenizer of a TikZero adapter (None: captions are refused)
        self.mode, self.preprocess = mode, preprocess
        self._cond = None                   # ((image key, caption), features) of the last conditioned side
        self.reset()

    def __str__(self):
        return self.__class__.__name__ + f" ({self.mode.upper().replace('_', '-')})"

    @classmethod
    def from_detikzify(cls, model, processor, mode=None, *args, **kwargs):
        from ..util.generation import unwrap_processor
        kwargs.pop("sync_on_compute", None)
        mode = getattr(model.config, "pooling_mode", "emd") if mode is None else mode
        tokenizer = processor.tokenizer if hasattr(model, "adapter") and hasattr(processor, "processor") else None
        return cls(model=model.model.vision_model, processor=unwrap_processor(processor).image_processor, mode=mode,
                   tokenizer=tokenizer, **kwargs)

    def _features(self, out) -> torch.Tensor:
        if self.mode == "cos":
            return out.pooler_output.squeeze()
        if self.mode == "cos_avg":
            return out.last_hidden_state.squeeze().mean(dim=0)
        return out.last_hidden_state.squeeze()

    def get_vision_features(self, image: Optional[Union[Image.Image, str]] = None, text: Optional[str] = None) -> torch.Tensor:
        if image is None and text is None:
            raise ValueError("either an image or a text is needed")
        if image is not None:
            image = load(image)
            if self.preprocess:
                image = expand(image, max(image.size), do_trim=True)
        if text is None:
            with torch.inference_mode():
                pixel_values = self.processor(images=image, return_tensors="pt")["pixel_values"]
                return self._features(self.model(pixel_values=pixel_values))
        if self.tokenizer is None:
            raise ValueError("a caption needs an ImageSim built (from_detikzify) from a model with a loaded TikZero adapter")
        key = (None if image is None else (image.size, hash(image.tobytes())), text)
        if self._cond is not None and self._cond[0] == key:
            return self._cond[1]
        with torch.inference_mode():
            enc = self.tokenizer(text=[text], truncation=True, return_tensors="pt")
            pixel_values = self.processor(images=image, return_tensors="pt")["pixel_values"] if image is not None else None
            feats = self._features(self.model(pixel_values=pixel_values, adapter_input_ids=enc["input_ids"],
                                              adapter_attention_mask=enc["attention_mask"]))
        self._cond = (key, feats)
        return feats

    @staticmethod
    def _emd_similarity(f1: torch.Tensor, f2: torch.Tensor) -> float:
        """2 tanh(-EMD) + 1 with EMD between the uniform distributions over the rows of f1 / f2, cost 1 - cosine (fp64)."""
        from math import tanh
        from scipy.optimize import linear_sum_assignment
        if f1.shape != f2.shape:
            raise ValueError(f"emd mode needs equally many patch tokens, got {tuple(f1.shape)} and {tuple(f2.shape)}")
        a = F.normalize(f1.double(), dim=1, eps=0.0)
        b = F.normalize(f2.double(), dim=1, eps=0.0)
        dists = (1.0 - a @ b.T).cpu().numpy()
        rows, cols = linear_sum_assignment(dists)
        return 2 * tanh(-float(dists[rows, cols].sum()) / dists.shape[0]) + 1

    def get_similarity(self, img1=None, img2=None, text1=None, text2=None, **_) -> float:
        f1, f2 = self.get_vision_features(img1, text1), self.get_vision_features(img2, text2)
        if f1.ndim > 1:
            return self._emd_similarity(f1, f2)
        return F.cosine_similarity(f1.double(), f2.double(), dim=0).item()

    def get_similarities(self, candidates: List[Union[Image.Image, str]], reference: Optional[Union[Image.Image, str]],
                         text: Optional[str] = None) -> List[float]:
        """SelfSim of several candidate renders against one reference figure: all images go through ONE batched ViT pass
        (the renders of a batch of parallel MCTS rollouts), the fp64 cosines are taken on the device and read back with a
        single transfer. Same values as ``get_similarity`` per pair (reference evaluate/imagesim.py:91-125). With ``text``
        (TikZero) the reference side (``reference`` or no image, plus the caption) is encoded by the adapted tower, once per
        (figure, caption), and the batch holds the candidates only."""
        target = None
        if text is not None:
            target = self.get_vision_features(reference, text)
        images = []
        for image in ([] if target is not None else [reference]) + list(candidates):
            image = load(image)
            if self.preprocess:
                image = expand(image, max(image.size), do_trim=True)
            images.append(image)
        owner = getattr(self.model, "_owner", None)
        with torch.inference_mode():
            if owner is not None and owner.device.type == "cuda" and hasattr(self.processor, "preprocess_device"):
                # resize + normalise on the device (bit-identical to the PIL path), straight into the ViT batch
                with owner._lock, owner._on_stream():
                    pixel_values = self.processor.preprocess_device(images, owner.engine)
                    owner._sync()
            else:
                pixel_values = torch.cat([self.processor(images=im, return_tensors="pt")["pixel_values"] for im in images])
            out = self.model(pixel_values=pixel_values)
            if self.mode == "emd":
                tokens = out.last_hidden_state
                if target is not None:
                    return [self._emd_similarity(tokens[i], target) for i in range(tokens.shape[0])]
                return [self._emd_similarity(tokens[i], tokens[0]) for i in range(1, tokens.shape[0])]
            feats = out.pooler_output if self.mode == "cos" else out.last_hidden_state.mean(dim=1)
            feats = feats.double()
            if target is not None:
                return F.cosine_similarity(feats, target.double()[None].expand_as(feats), dim=1).tolist()
            return F.cosine_similarity(feats[1:], feats[:1].expand_as(feats[1:]), dim=1).tolist()

    def update(self, img1=None, img2=None, text1=None, text2=None):
        """reference imagesim.py:127-142: each side needs an image or a text; lists pair up element-wise."""
        inputs = {}
        for key, value in dict(img1=img1, img2=img2, text1=text1, text2=text2).items():
            if value is not None:
                inputs[key] = value if isinstance(value, list) else [value]
        if {"img1", "text1"}.isdisjoint(inputs) or {"img2", "text2"}.isdisjoint(inputs):
            raise ValueError("each side of the comparison needs an image or a text")
        if len(set(map(len, inputs.values()))) != 1:
            raise ValueError("img1 / img2 / text1 / text2 lists must have the same length")
        for values in zip(*inputs.values()):
            self.score += self.get_similarity(**dict(zip(inputs.keys(), values)))
            self.n_samples += 1

    def compute(self) -> float:
        return self.score / self.n_samples

    def reset(self):
        self.score, self.n_samples = 0.0, 0
