"""Shared builders for the GPU parity tests / smoke / bench: product modules loaded with the
oracle's seeded weights."""
import os

import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "configs")


def _load(mod, sd, device):
    mod.load_state_dict(sd, strict=True, assign=True)
    return mod.to(device).eval()


def build_g(sd, device="cuda"):
    from megatts2_b200.models.megatts2 import MegaG
    with torch.device("meta"):
        g = MegaG.from_hparams(os.path.join(CFG, "config_gan.yaml"))
    return _load(g, sd, device)


def build_plm(sd, device="cuda"):
    from megatts2_b200.utils.utils import instantiate_class
    with torch.device("meta"):
        m = instantiate_class((), yaml.safe_load(open(os.path.join(CFG, "config_plm.yaml")))["model"]["plm"])
    return _load(m, sd, device)


def build_adm(sd, device="cuda"):
    from megatts2_b200.utils.utils import instantiate_class
    with torch.device("meta"):
        m = instantiate_class((), yaml.safe_load(open(os.path.join(CFG, "config_adm.yaml")))["model"]["adm"])
    return _load(m, sd, device)


def build_hifigan(sd, device="cuda"):
    from megatts2_b200.models.megatts2 import HIFIGAN, HifiganGenerator
    with torch.device("meta"):
        gen = HifiganGenerator()
    return HIFIGAN(_load(gen, sd, device)).eval()


def build_megatts(wg, wp, wa, wh, device="cuda"):
    from megatts2_b200.models.megatts2 import Megatts
    return Megatts(generator=build_g(wg, device), plm=build_plm(wp, device), adm=build_adm(wa, device),
                   hifi_gan=build_hifigan(wh, device), device=device)


def record(name, payload):
    """Append a measured parity figure to the JSON-lines file named by $MEGATTS2_PARITY_LOG (nothing when it is unset:
    the tests never write into the source tree)."""
    import json
    path = os.environ.get("MEGATTS2_PARITY_LOG")
    if not path:
        return
    with open(path, "a") as f:
        f.write(json.dumps({"name": name, **payload}) + "\n")
