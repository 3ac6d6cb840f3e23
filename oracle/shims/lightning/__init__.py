"""Stand-in for `import lightning as L` in models/modules/utils.py: only `L.LightningModule` is referenced."""
import torch


class LightningModule(torch.nn.Module):
    def save_hyperparameters(self, *args, **kwargs):
        pass

    @classmethod
    def load_from_checkpoint(cls, checkpoint_path, **kwargs):
        """A freshly constructed module; oracle/faed.py loads the seeded weights into it afterwards."""
        return cls(**kwargs)
