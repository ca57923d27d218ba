"""sivo_b200 -- H100-native (sm_90a) SIVO perception front-end (Bayesian SegNet MC-dropout + ORB extractor).
Host-side mirrors of the reference's two operators over the C-ABI of libsivo_b200.so."""
from .segnet import BayesianSegNet, BayesianSegNetParams  # noqa: F401
from .orb import ORBextractor, distribute_octtree, stereo_hamming, stereo_match, KP_DTYPE  # noqa: F401
