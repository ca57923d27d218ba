"""sivo_b200 -- H100-native (sm_90a) SIVO perception front-end (Bayesian SegNet MC-dropout + ORB extractor).
Host-side mirrors of the reference's two operators over the C-ABI of libsivo_b200.so."""
from .segnet import BayesianSegNet, BayesianSegNetParams, sample_ranges  # noqa: F401
from .orb import ORBextractor, distribute_octtree, stereo_hamming, stereo_match, stereo_match_device, KP_DTYPE  # noqa: F401
from .info import InfoCamera, info_select, info_select_device, make_camera  # noqa: F401
from .track import (MAP_POINT_DTYPE, TrackFrame, make_frame, map_points, search_last_frame, search_last_frame_device,  # noqa: F401
                    search_local_points, search_local_points_device)
from .pose import PoseResult, pose_gather_device, pose_optimize, pose_optimize_device  # noqa: F401
from .bow import Vocabulary, compute_bow, compute_bow_device, search_by_bow, search_by_bow_device  # noqa: F401
from .reloc import PnpSolver  # noqa: F401
