"""Stand-in for the reference's models/pano/PanoGenerator.py as EvalPanoGen uses it: PanoBase with its default
hyperparameters (no prompt prefixes, per-view prompts from batch['prompt']), save_hyperparameters reading the caller's
arguments, and a trainer whose batch_to_device is the identity (everything stays on the CPU)."""
import inspect
import types

from models.modules.utils import WandbLightningModule


class PanoBase(WandbLightningModule):
    def __init__(self, **kwargs):
        super().__init__()
        self.hparams = types.SimpleNamespace(pano_prompt_prefix="", pers_prompt_prefix="", mv_pano_prompt=False,
                                             copy_pano_prompt=False, **kwargs)
        self.trainer = types.SimpleNamespace(strategy=types.SimpleNamespace(batch_to_device=lambda b: b))

    def save_hyperparameters(self):
        for k, v in inspect.currentframe().f_back.f_locals.items():
            if k not in ("self", "kwargs", "__class__"):
                setattr(self.hparams, k, v)

    def get_pano_prompt(self, batch):
        return list(batch["pano_prompt"])

    def get_pers_prompt(self, batch):
        # batch['prompt'] is collated view-major (one sequence per view, over the batch): panorama-major order here
        return [p for per_pano in zip(*batch["prompt"]) for p in per_pano]
