"""sys.modules shims so the REAL reference (a checkout named by $MEGATTS2_REFERENCE) imports here.

Fixture-generation infrastructure only (oracle/make_golden.py); the tests never need the reference.
The reference imports matplotlib, pypinyin, phonemizer, lhotse, speechbrain,
librosa, lightning and tqdm at module import time (utils/utils.py:5,
modules/tokenizer.py:1-17, models/megatts2.py:18-25, modules/datamodule.py:1-21);
none of them is on the synthesis hot path except the two speechbrain pieces,
which are bound to restatements here.
"""
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("MEGATTS2_REFERENCE", "")


def reference_available() -> bool:
    return bool(REFERENCE_ROOT) and os.path.isdir(os.path.join(REFERENCE_ROOT, "modules"))


def _mod(name, **attrs):
    m = types.ModuleType(name)
    m.__path__ = []
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def _torchaudio_mel_spectogram(sample_rate, hop_length, win_length, n_fft, n_mels,
                               f_min, f_max, power, normalized, min_max_energy_norm,
                               norm, mel_scale, compression, audio):
    """speechbrain.lobes.models.FastSpeech2.mel_spectogram, restated [memory]:
    torchaudio MelSpectrogram with the given kwargs, then log(clamp(., 1e-5)).
    Returns (mel, rmse); the reference discards the second value
    (modules/tokenizer.py:108)."""
    import torch
    import torchaudio
    tr = torchaudio.transforms.MelSpectrogram(
        sample_rate=sample_rate, hop_length=hop_length, win_length=win_length,
        n_fft=n_fft, n_mels=n_mels, f_min=f_min, f_max=f_max, power=power,
        normalized=normalized, norm=norm, mel_scale=mel_scale)
    mel = tr(audio)
    rmse = torch.norm(mel, dim=0)
    if compression:
        mel = torch.log(torch.clamp(mel, min=1e-5))
    return mel, rmse


class _StubHIFIGAN:
    """speechbrain.pretrained.HIFIGAN stand-in wrapping the oracle generator."""

    def __init__(self, sd):
        self.sd = sd

    @classmethod
    def from_hparams(cls, source=None, **kw):
        from . import weights
        return cls(weights.hifigan_state_dict())

    def eval(self):
        return self

    def decode_batch(self, mel):
        from . import ref_megatts2 as R
        return R.hifigan_decode_batch(self.sd, mel)


def install():
    """Install the shims and put the reference on sys.path. Idempotent."""
    if not reference_available():
        raise RuntimeError("reference tree not present at %s" % REFERENCE_ROOT)
    if "speechbrain.pretrained" in sys.modules and getattr(
            sys.modules["speechbrain.pretrained"], "_mtts_stub", False):
        return
    import torch.nn as nn

    class _Any:
        def __init__(self, *a, **k):
            pass

        def __call__(self, *a, **k):
            return self

    _mod("matplotlib")
    _mod("matplotlib.pyplot", Figure=object)
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    _mod("pypinyin", pinyin=_Any(), Style=_Any())
    _mod("phonemizer")
    _mod("phonemizer.separator", Separator=_Any)
    _mod("lhotse", CutSet=type("CutSet", (), {}), load_manifest=_Any())
    _mod("lhotse.features", FeatureExtractor=type("FeatureExtractor", (), {}))
    _mod("lhotse.utils", Seconds=float, compute_num_frames=_Any())
    _mod("lhotse.dataset", DynamicBucketingSampler=_Any, SimpleCutSampler=_Any)
    _mod("lhotse.dataset.collation", collate_features=_Any())
    _mod("lhotse.dataset.input_strategies", _get_executor=_Any())
    _mod("speechbrain")
    _mod("speechbrain.lobes")
    _mod("speechbrain.lobes.models")
    _mod("speechbrain.lobes.models.FastSpeech2", mel_spectogram=_torchaudio_mel_spectogram)
    sb = _mod("speechbrain.pretrained", HIFIGAN=_StubHIFIGAN)
    sb._mtts_stub = True
    _mod("librosa")
    _mod("lightning")
    _mod("lightning.pytorch", LightningModule=nn.Module,
         LightningDataModule=type("LightningDataModule", (), {}))
    sys.modules["lightning"].pytorch = sys.modules["lightning.pytorch"]
    if "tqdm" not in sys.modules:
        try:
            import tqdm  # noqa: F401
            import tqdm.auto  # noqa: F401
        except Exception:
            _mod("tqdm", tqdm=_Any())
            _mod("tqdm.auto", tqdm=_Any())
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)


def build_reference_models():
    """Instantiate the real reference MegaG / MegaPLM / MegaADM from its YAMLs
    (models/megatts2.py:86-104, utils/utils.py:86-102).  Weights are whatever
    the constructors produce; callers load oracle.weights state dicts."""
    install()
    import warnings
    import yaml
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from models.megatts2 import MegaG  # type: ignore
        from utils.utils import instantiate_class  # type: ignore
    cfg = os.path.join(REFERENCE_ROOT, "configs")
    G = MegaG.from_hparams(os.path.join(cfg, "config_gan.yaml"))
    with open(os.path.join(cfg, "config_plm.yaml")) as f:
        plm = instantiate_class((), yaml.safe_load(f)["model"]["plm"])
    with open(os.path.join(cfg, "config_adm.yaml")) as f:
        adm = instantiate_class((), yaml.safe_load(f)["model"]["adm"])
    return G.eval(), plm.eval(), adm.eval()
