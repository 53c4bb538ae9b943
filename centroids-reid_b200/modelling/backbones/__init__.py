"""ResNet50 / ResNet50-IBN-A trunks: reference-layout parameters + the H100 inference engine."""
