"""Stand-in for `import wandb` in models/modules/utils.py; nothing from it is called by the FAED encoder or metric."""
