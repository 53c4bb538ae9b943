"""centroids-reid_b200 -- H100-native engine for the centroid-triplet re-ID hot path
(embedding forward -> CTL / center / CE losses -> query x gallery retrieval and CMC / mAP) of
mikwieczorek/centroids-reid, behind the reference's own module surface:

    losses.triplet_loss   TripletLoss, euclidean_dist, cosine_dist, hard_example_mining,
                          CrossEntropyLabelSmooth          (losses/triplet_loss.py)
    losses.center_loss    CenterLoss                       (losses/center_loss.py)
    utils.reid_metric     get_euclidean, get_cosine, get_dist_func, R1_mAP
    utils.eval_reid       eval_func
    modelling.*           Baseline, CTL step, base-model step (modelling/, train_ctl_model.py, train_base_model.py)
    inference.*           run_inference, calculate_centroids, get_similar

The directory name carries a hyphen (it is mandated by the build contract), so import it as
``importlib.import_module("centroids-reid_b200")`` or through the ``ctl_b200`` alias module
at the repository root.  All arithmetic runs in hand-written sm_90a CUDA reached through
the C ABI of ``libctl_b200.so`` (include/ctl_b200.h); there is no CPU fallback.
"""
__version__ = "0.1.0"

from . import _native  # noqa: F401
