"""
Drop-in boundary (SURVEY.md §8b): the REFERENCE's own inference driver — detikzify/infer/generate.py (DetikzifyGenerator,
DetikzifyPipeline, WideNode, rollout streaming), detikzify/mcts/*, detikzify/util/{functools,generation}.py, byte-compiled
into oracle/_ref by oracle/build_ref.py and executed unmodified — runs on top of the objects ``detikzify_b200`` returns (model with ``generate``,
processor, tokenizer), with a scripted engine standing in for the GPU. This is the claim "only the ``load`` import changes".

Stubbed because they are absent offline and outside the path: torchmetrics (base class only), the TeX toolchain
(``infer/tikz.py``: pdf2image / pdfCropMargins / pymupdf → a TikzDocument that "compiles" everything), ``util/image.py``
(pymupdf, requests → two small PIL helpers), ``model/adapter`` (``has_adapter`` → False), POT's ``emd2`` (v1 models pool
with "cos"). The reference's ``evaluate/imagesim.py`` (SelfSim reward) is loaded for real on a minimal ``torchmetrics.Metric``.
Skipped where oracle/_ref was not built (no reference checkout at build time) or was built by another Python version.
The two tests that compare NUMBERS with the reference (image preprocessing, EMD SelfSim) run everywhere: they compare with
tests/golden/reference_dropin.npz, which tests/golden/make_reference_dropin_golden.py stored from the reference's own code.
"""
import contextlib
import importlib.util
import os
import sys
import types

import pytest
import torch
from PIL import Image, ImageDraw

from scripted_engine import ScriptedEngine

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "detikzify")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_dropin.npz")


def _ref_usable():
    """oracle/_ref exists and its byte code was compiled by this interpreter version."""
    probe = os.path.join(REF, "mcts", "node.pyc")
    if not os.path.isfile(probe):
        return False
    with open(probe, "rb") as f:
        return f.read(4) == importlib.util.MAGIC_NUMBER


needs_ref = pytest.mark.skipif(not _ref_usable(), reason="oracle/_ref was not built for this Python (no reference checkout at build time)")


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


@contextlib.contextmanager
def reference_modules():
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] in ("torchmetrics", "ot", "detikzify")}
    for k in list(saved):
        del sys.modules[k]
    try:
        tm = types.ModuleType("torchmetrics")
        tm.Metric = type("Metric", (), {})
        sys.modules["torchmetrics"] = tm
        for pkg in ("detikzify", "detikzify.infer", "detikzify.mcts", "detikzify.util", "detikzify.model", "detikzify.evaluate"):
            m = types.ModuleType(pkg)
            m.__path__ = []
            sys.modules[pkg] = m
        # real reference modules
        _load("detikzify.mcts.node", f"{REF}/mcts/node.pyc")
        _load("detikzify.mcts.montecarlo", f"{REF}/mcts/montecarlo.pyc")
        fn = _load("detikzify.util.functools", f"{REF}/util/functools.pyc")
        gn = _load("detikzify.util.generation", f"{REF}/util/generation.pyc")
        util = sys.modules["detikzify.util"]
        for mod in (fn, gn):
            for k, v in vars(mod).items():
                if not k.startswith("_"):
                    setattr(util, k, v)
        util.load = lambda image: image.convert("RGB") if isinstance(image, Image.Image) else Image.open(image).convert("RGB")

        def expand(image, size, do_trim=False):
            canvas = Image.new("RGB", (size, size), "white")
            canvas.paste(image, ((size - image.width) // 2, (size - image.height) // 2))
            return canvas
        util.expand = expand
        # stubs for what is absent offline / outside the path
        adapter = types.ModuleType("detikzify.model.adapter")
        adapter.has_adapter = lambda model: False
        sys.modules[adapter.__name__] = adapter
        adapter.AdapterProcessor = type("AdapterProcessor", (), {})
        adapter.CrossAttentionAdapterMixin = type("CrossAttentionAdapterMixin", (), {})
        _load("detikzify.util.torch", f"{REF}/util/torch.pyc")
        util.infer_device = sys.modules["detikzify.util.torch"].infer_device
        # torchmetrics.Metric: the slice of its protocol the reference's ImageSim relies on (states, reset, device/dtype)
        class Metric(torch.nn.Module):
            def __init__(self, **kwargs):
                super().__init__()
                self._defaults, self._dtype = {}, torch.float32

            def add_state(self, name, default, dist_reduce_fx=None):
                self._defaults[name] = default
                setattr(self, name, default.clone())

            def reset(self):
                for k, v in self._defaults.items():
                    setattr(self, k, v.clone())

            def set_dtype(self, dtype):
                self._dtype = dtype
                return self

            device = property(lambda self: self._device)
            dtype = property(lambda self: self._dtype)
        tm.Metric = Metric
        tmf = types.ModuleType("torchmetrics.functional")
        tmf.pairwise_cosine_similarity = lambda a, b: torch.nn.functional.normalize(a, dim=-1) @ torch.nn.functional.normalize(b, dim=-1).T
        sys.modules["torchmetrics.functional"] = tmf
        ot, otlp = types.ModuleType("ot"), types.ModuleType("ot.lp")
        def emd2(M, a, b):   # POT's ot.lp.emd2 (absent offline) restated: the transport LP, empty marginals = uniform
            import numpy as np
            from scipy.optimize import linprog
            M = np.asarray(M, dtype=np.float64)
            n, m = M.shape
            a = np.full(n, 1.0 / n) if len(a) == 0 else np.asarray(a, dtype=np.float64)
            b = np.full(m, 1.0 / m) if len(b) == 0 else np.asarray(b, dtype=np.float64)
            A_eq = np.zeros((n + m, n * m))
            for i in range(n):
                A_eq[i, i * m:(i + 1) * m] = 1.0
            for j in range(m):
                A_eq[n + j, j::m] = 1.0
            res = linprog(M.reshape(-1), A_eq=A_eq, b_eq=np.concatenate([a, b]), bounds=(0, None), method="highs")
            assert res.status == 0, res.message
            return float(res.fun)
        otlp.emd2 = emd2
        sys.modules["ot"], sys.modules["ot.lp"] = ot, otlp
        _load("detikzify.evaluate.imagesim", f"{REF}/evaluate/imagesim.pyc")
        tikz = types.ModuleType("detikzify.infer.tikz")

        class TikzDocument:
            """Stand-in for the TeX toolchain: every program 'compiles'."""
            def __init__(self, code, timeout=None):
                self.code, self.timeout = code, timeout
            is_rasterizable = True
            compiled_with_errors = False
            errors = {}

            def rasterize(self):
                return Image.new("RGB", (32, 32), "white")
        tikz.TikzDocument = TikzDocument
        sys.modules[tikz.__name__] = tikz
        yield _load("detikzify.infer.generate", f"{REF}/infer/generate.pyc")
    finally:
        for k in [k for k in sys.modules if k.split(".")[0] in ("torchmetrics", "ot", "detikzify")]:
            del sys.modules[k]
        sys.modules.update(saved)


@pytest.fixture()
def reference_infer():
    with reference_modules() as mod:
        yield mod


def _ours(eos_at=40):
    from detikzify_b200.model import build_processor, preset
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    cfg = preset("tiny")
    eng = ScriptedEngine(cfg, eos_at=eos_at)
    return DetikzifyForCausalLM(cfg, engine=eng), build_processor(cfg), eng


def _figure(size=90):
    im = Image.new("RGB", (size, size + 20), "white")
    d = ImageDraw.Draw(im)
    d.line((10, 10, size - 10, size - 5), fill="black", width=3)
    d.ellipse((20, 30, 50, 60), outline="black")
    return im


@needs_ref
def test_reference_pipeline_sample_runs_on_our_model(reference_infer):
    model, proc, eng = _ours(eos_at=30)
    pipe = reference_infer.DetikzifyPipeline(model=model, processor=proc, metric="fast")
    assert pipe.gen_kwargs["max_length"] == proc.tokenizer.model_max_length and pipe.gen_kwargs["do_sample"] is True
    doc = pipe.sample(image=_figure())
    assert isinstance(doc.code, str) and len(doc.code) > 0
    # the reference passed its own generation kwargs straight into our generate() (infer/generate.py:218-227)
    kw = eng.last_sampling
    assert kw["bad_token"] == model.config.image_token_id and kw["begin_suppress_token"] == model.config.text_config.eos_token_id
    assert kw["do_sample"] and abs(kw["temperature"] - 0.8) < 1e-6 and abs(kw["top_p"] - 0.95) < 1e-6


@needs_ref
def test_reference_mcts_simulate_runs_on_our_model(reference_infer):
    model, proc, eng = _ours(eos_at=36)
    pipe = reference_infer.DetikzifyPipeline(model=model, processor=proc, metric="fast")
    results = list(pipe.simulate(image=_figure(), expansions=4))
    assert len(results) == 4
    for score, doc in results:
        assert score == 1 and isinstance(doc.code, str)          # scorable - compiled_with_errors with the stub compiler
    # rollouts went through the reference's ThreadPool + TokenStreamer + stopping-criteria path and our streaming contract
    assert sum(1 for c in eng.calls if c[0] == "gen_begin") >= 4


@needs_ref
def test_reference_generator_abort_and_tree(reference_infer):
    model, proc, eng = _ours(eos_at=60)
    gen = reference_infer.DetikzifyGenerator(model=model, processor=proc, image=_figure(), metric=None,
                                             max_length=proc.tokenizer.model_max_length, temperature=0.8, top_p=0.95, top_k=0,
                                             do_sample=True)
    out = [next(gen.simulate(expansions=1)) for _ in range(2)]
    root = gen.montecarlo.root_node
    assert root.visits >= 2 and root.children and root.children[0].is_widen_node
    assert all(score == 1 for score, _ in out)
    # newline bookkeeping of the reference works with our tokenizer (vocab / decode protocol)
    assert gen.newlineinfo and all(v.num_lines >= 1 for v in gen.newlineinfo.values())


@needs_ref
def test_reference_selfsim_metric_runs_on_our_vision_model(reference_infer):
    """metric="model": the reference's ImageSim.from_detikzify wraps OUR model.model.vision_model / image processor and
    computes the SelfSim reward from pooler_output (evaluate/imagesim.py:60-125); MCTS then min-max-normalises it."""
    model, proc, eng = _ours(eos_at=36)
    pipe = reference_infer.DetikzifyPipeline(model=model, processor=proc, metric="model")
    assert type(pipe.metric).__name__ == "ImageSim" and pipe.metric.mode == "cos"
    pipe.metric.update(img1=_figure(), img2=_figure())
    assert pipe.metric.compute() == pytest.approx(1.0)            # identical figures -> cosine 1
    pipe.metric.reset()
    results = list(pipe.simulate(image=_figure(), expansions=3))
    assert len(results) == 3 and all(-1.0 <= score <= 1.0 + 1e-9 for score, _ in results)
    assert any(c[0] == "vit_encode" for c in eng.calls)


def _other_figure():
    other = Image.new("RGB", (80, 80), "white")
    ImageDraw.Draw(other).ellipse((10, 10, 60, 70), outline="black", width=4)
    return other


def _preprocess_images():
    import numpy as np
    rng = np.random.default_rng(3)
    return [_figure(90), _figure(384).resize((384, 384)), Image.fromarray(rng.integers(0, 255, (200, 311, 3), dtype=np.uint8))]


def _pixel_sample(n):
    """Fixed, seeded sample of the 3 x 384 x 384 pixel values (the golden file stores these positions only)."""
    import numpy as np
    return np.random.default_rng(11).choice(3 * 384 * 384, size=n, replace=False)


def reference_emd_case():
    """Runs the REFERENCE's ImageSim in "emd" mode on our vision model -> (patch tokens of both figures, its similarities)."""
    with reference_modules():
        RefImageSim = sys.modules["detikzify.evaluate.imagesim"].ImageSim
        model, proc, _ = _ours(eos_at=36)
        ref = RefImageSim.from_detikzify(model, proc, mode="emd")
        f1, f2 = ref.get_vision_features(_figure()), ref.get_vision_features(_other_figure())
        return f1, f2, ref.get_similarity(_figure(), _other_figure()), ref.get_similarity(_figure(), _figure())


def reference_preprocess_case():
    """Runs the REFERENCE's DetikzifyImageProcessor (only ``timm.data`` / ``timm.models``, which its ``from_pretrained`` would
    consult for the SigLIP data config, are stubbed with timm's published config of vit_so400m_patch14_siglip_384:
    input 3x384x384, mean = std = 0.5, bicubic) -> (its attributes, pixel_values per test image)."""
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] == "timm"}
    try:
        timm = types.ModuleType("timm"); timm.__path__ = []
        data, models = types.ModuleType("timm.data"), types.ModuleType("timm.models")
        cfg = {"input_size": [3, 384, 384], "mean": (0.5, 0.5, 0.5), "std": (0.5, 0.5, 0.5), "crop_mode": "center"}
        models.resolve_pretrained_cfg = lambda variant: types.SimpleNamespace(to_dict=lambda: dict(cfg))
        data.resolve_data_config = lambda d: dict(d)
        sys.modules.update({"timm": timm, "timm.data": data, "timm.models": models})
        ref_mod = _load("ref_processing_detikzify", f"{REF}/model/v1/processing_detikzify.pyc")
        ref = ref_mod.DetikzifyImageProcessor.from_pretrained("vit_so400m_patch14_siglip_384.webli")
    finally:
        for k in [k for k in sys.modules if k.split(".")[0] == "timm"]:
            del sys.modules[k]
        sys.modules.update(saved)
        sys.modules.pop("ref_processing_detikzify", None)
    attrs = [float(ref.size["height"]), float(ref.size["width"]), *map(float, ref.image_mean), *map(float, ref.image_std),
             float(int(ref.resample)), float(ref.rescale_factor)]
    return attrs, [ref(images=im, return_tensors="pt")["pixel_values"].float() for im in _preprocess_images()]


def test_reference_emd_selfsim_agrees_with_ours():
    """The v2 default reward: the reference's own ImageSim in "emd" mode (evaluate/imagesim.py:105-107,121-123; POT's emd2
    restated as the transport LP) and ours (assignment solver) on the same vision model object and image processor. The
    reference side is stored (patch tokens it extracted and the similarities it computed) and re-run live where oracle/_ref
    is available."""
    import numpy as np
    from detikzify_b200.evaluate.imagesim import ImageSim as Ours
    g = np.load(GOLDEN)
    cases = [(torch.from_numpy(g["emd_f1"]), torch.from_numpy(g["emd_f2"]), float(g["emd_sim"]), float(g["emd_self"]))]
    if _ref_usable():
        cases.append(reference_emd_case())
    model, proc, eng = _ours(eos_at=36)
    ours = Ours.from_detikzify(model, proc, mode="emd")
    for f1, f2, a, a_self in cases:
        # the reference object feeds bf16 pixels (its .to(device, dtype)), ours fp32: compare the solvers on the SAME patch tokens ...
        assert f1.ndim == 2 and a == pytest.approx(Ours._emd_similarity(f1.float(), f2.float()), abs=1e-9) and -1.0 < a < 1.0
        # ... and the two end-to-end paths within the bf16 rounding of the inputs
        assert a == pytest.approx(ours.get_similarity(_figure(), _other_figure()), abs=5e-2)
        assert a_self == pytest.approx(1.0, abs=1e-9)


def test_image_processor_matches_reference_preprocess():
    """§8 row a1: our host-side DetikzifyImageProcessor against the reference's own class
    (detikzify/model/v1/processing_detikzify.py:162-253): its attributes and a fixed sample of 60 000 of the pixel values it
    produced per test image are stored; where oracle/_ref is available the class is also run live on every pixel."""
    import numpy as np
    from detikzify_b200.model.processing import DetikzifyImageProcessor
    ours = DetikzifyImageProcessor(size=384)
    mine = [float(ours.size["height"]), float(ours.size["width"]), *ours.image_mean, *ours.image_std, float(ours.resample), ours.rescale_factor]
    g = np.load(GOLDEN)
    assert np.allclose(g["proc_attrs"], mine, rtol=0, atol=1e-12) and ours.resample == 3
    idx = _pixel_sample(g["proc_pixels"].shape[1])
    outs = [ours(im, return_tensors="pt")["pixel_values"] for im in _preprocess_images()]
    for b, want in zip(outs, g["proc_pixels"]):
        assert b.shape == (1, 3, 384, 384) and b.dtype == torch.float32
        assert np.abs(b.reshape(-1).numpy()[idx] - want).max() < 1e-6
    if _ref_usable():
        attrs, ref_outs = reference_preprocess_case()
        assert np.allclose(attrs, mine, rtol=0, atol=1e-12)
        for a, b in zip(ref_outs, outs):
            assert a.shape == b.shape and (a - b).abs().max().item() < 1e-6
