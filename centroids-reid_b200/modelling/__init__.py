"""Drop-ins for the reference's modelling/ package (backbones, Baseline, CTL and base-model steps)."""
