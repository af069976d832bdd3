from .ape_rpe import ape, rpe
