"""Make the UNMODIFIED reference scripts run on the H100 modules.

    import rq_vae_recommender_b200.dropin as dropin
    dropin.install(reference_root="/path/to/RQ-VAE-Recommender")   # before `import train_rqvae`
    import train_rqvae; train_rqvae.train(...)

``install`` pre-seeds ``sys.modules`` so that every ``from modules.quantize import ...`` / ``from init.kmeans import
...`` inside the reference (train_rqvae.py:13-15, modules/tokenizer/semids.py:10, train_decoder.py:13-20) resolves to
the replacement modules of this package; everything else (data/, evaluate/, the scripts) is imported from the reference
tree untouched.  ``replace_model=True`` also aliases ``modules.model`` (train_decoder.py:14), whose
``EncoderDecoderRetrievalModel.generate`` then runs its beam search on the fused sampling and selection kernel;
``search="beam"`` (with ``replace_model=True``) makes the exhaustive, deterministic beam search over every code its default, so
an unmodified ``train_decoder.py`` evaluates with it (``search="exact"``: the exact top-k search, the most probable corpus tuples
with no search error); ``decoder="fused"`` (with ``replace_model=True``) likewise makes generate's
decoder passes run on the fused decoder-step kernels (``FusedT5Decode``), and ``encoder="fused"`` its encoder pass over the
unpadded positions only (``FusedT5Encode``); ``forward_encoder="fused"`` makes the training pass ``forward`` run its encoder on
the trainable packed pass (``FusedT5EncodeTrain``), and ``forward_decoder="fused"`` its decoder on the fused training
decoder (``FusedT5DecodeTrain``).  ``encoder_attention="tf32"`` makes the fused encoder passes (of ``generate`` and
``forward``) run their self-attention on the TF32 tensor-core kernels.  ``exclude_history=True`` (with ``replace_model=True``)
makes ``generate_next_sem_id``, ``generate_items`` and ``rank_items`` leave each history's own items out by default, so an
unmodified ``train_decoder.py`` evaluates with seen items masked.  ``replace_metrics=True`` also aliases ``evaluate.metrics``
(train_decoder.py:13), whose ``TopKAccumulator`` accumulates on the device without waiting on the host.  Checkpoints pickle ``modules.quantize.Quantize`` etc. by module path,
so ``torch.load(..., weights_only=False)`` of the shipped files also lands on the replacement classes.
gin-config is not in this image: a small compatible shim is registered as ``gin`` when the real one is missing.
"""
import importlib
import sys
import types

_ALIASES = {
    "modules.quantize": "rq_vae_recommender_b200.modules.quantize",
    "modules.rqvae": "rq_vae_recommender_b200.modules.rqvae",
    "modules.encoder": "rq_vae_recommender_b200.modules.encoder",
    "modules.loss": "rq_vae_recommender_b200.modules.loss",
    "modules.normalize": "rq_vae_recommender_b200.modules.normalize",
    "init.kmeans": "rq_vae_recommender_b200.init.kmeans",
    "distributions.gumbel": "rq_vae_recommender_b200.distributions.gumbel",
}
_TOKENIZER = ("modules.tokenizer.semids", "rq_vae_recommender_b200.modules.tokenizer.semids")
_MODEL = ("modules.model", "rq_vae_recommender_b200.modules.model")
_METRICS = ("evaluate.metrics", "rq_vae_recommender_b200.evaluate.metrics")


def install(reference_root=None, replace_tokenizer=True, gin_shim=True, replace_model=False, search="sample",
            replace_metrics=False, decoder="hf", encoder="hf", forward_encoder="hf", forward_decoder="hf",
            encoder_attention="fp32", exclude_history=False):
    if search not in ("sample", "beam", "exact"):
        raise ValueError(f"search must be 'sample', 'beam' or 'exact', got {search!r}")
    if search != "sample" and not replace_model:
        raise ValueError(f"search={search!r} selects the replacement model's search: it needs replace_model=True")
    if decoder not in ("hf", "fused"):
        raise ValueError(f"decoder must be 'hf' or 'fused', got {decoder!r}")
    if decoder != "hf" and not replace_model:
        raise ValueError(f"decoder={decoder!r} selects the replacement model's decoder passes: it needs replace_model=True")
    if encoder not in ("hf", "fused"):
        raise ValueError(f"encoder must be 'hf' or 'fused', got {encoder!r}")
    if encoder != "hf" and not replace_model:
        raise ValueError(f"encoder={encoder!r} selects the replacement model's encoder pass: it needs replace_model=True")
    if forward_encoder not in ("hf", "fused"):
        raise ValueError(f"forward_encoder must be 'hf' or 'fused', got {forward_encoder!r}")
    if forward_encoder != "hf" and not replace_model:
        raise ValueError(f"forward_encoder={forward_encoder!r} selects the replacement model's training encoder pass: it needs "
                         "replace_model=True")
    if forward_decoder not in ("hf", "fused"):
        raise ValueError(f"forward_decoder must be 'hf' or 'fused', got {forward_decoder!r}")
    if forward_decoder != "hf" and not replace_model:
        raise ValueError(f"forward_decoder={forward_decoder!r} selects the replacement model's training decoder pass: it needs "
                         "replace_model=True")
    if encoder_attention not in ("fp32", "tf32"):
        raise ValueError(f"encoder_attention must be 'fp32' or 'tf32', got {encoder_attention!r}")
    if encoder_attention != "fp32" and not replace_model:
        raise ValueError(f"encoder_attention={encoder_attention!r} selects the replacement model's fused encoder attention: it "
                         "needs replace_model=True")
    if exclude_history not in (False, True):
        raise ValueError(f"exclude_history must be True or False, got {exclude_history!r}")
    if exclude_history and not replace_model:
        raise ValueError("exclude_history=True selects the replacement model's exclusion of seen items: it needs replace_model=True")
    if gin_shim and "gin" not in sys.modules:
        try:
            import gin  # noqa: F401
        except ImportError:
            from . import gin_compat
            sys.modules["gin"] = gin_compat
    if reference_root is not None and reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    parents = ("init", "distributions") + (("evaluate",) if replace_metrics else ())
    for parent in parents:                             # namespace packages in the reference (no __init__.py)
        if parent not in sys.modules and reference_root is None:
            sys.modules[parent] = types.ModuleType(parent)
            sys.modules[parent].__path__ = []
    for alias, real in _ALIASES.items():
        sys.modules[alias] = importlib.import_module(real)
    if replace_tokenizer:
        sys.modules[_TOKENIZER[0]] = importlib.import_module(_TOKENIZER[1])
    if replace_model:
        sys.modules[_MODEL[0]] = importlib.import_module(_MODEL[1])
        sys.modules[_MODEL[0]].DEFAULT_SEARCH = search
        sys.modules[_MODEL[0]].DEFAULT_DECODER = decoder
        sys.modules[_MODEL[0]].DEFAULT_ENCODER = encoder
        sys.modules[_MODEL[0]].DEFAULT_FORWARD_ENCODER = forward_encoder
        sys.modules[_MODEL[0]].DEFAULT_FORWARD_DECODER = forward_decoder
        sys.modules[_MODEL[0]].DEFAULT_ENCODER_ATTENTION = encoder_attention
        sys.modules[_MODEL[0]].DEFAULT_EXCLUDE_HISTORY = exclude_history
    if replace_metrics:
        sys.modules[_METRICS[0]] = importlib.import_module(_METRICS[1])
    return sorted(list(_ALIASES) + ([_TOKENIZER[0]] if replace_tokenizer else []) + ([_MODEL[0]] if replace_model else [])
                  + ([_METRICS[0]] if replace_metrics else []))


def uninstall():
    for alias in list(_ALIASES) + [_TOKENIZER[0], _MODEL[0], _METRICS[0]]:
        mod = sys.modules.get(alias)
        if mod is not None and mod.__name__.startswith("rq_vae_recommender_b200"):
            del sys.modules[alias]
    model = sys.modules.get(_MODEL[1])
    if model is not None:
        model.DEFAULT_SEARCH = "sample"
        model.DEFAULT_DECODER = "hf"
        model.DEFAULT_ENCODER = "hf"
        model.DEFAULT_FORWARD_ENCODER = "hf"
        model.DEFAULT_FORWARD_DECODER = "hf"
        model.DEFAULT_ENCODER_ATTENTION = "fp32"
        model.DEFAULT_EXCLUDE_HISTORY = False
