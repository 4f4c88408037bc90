"""`from estimater import *` as run_demo.py:10 / run_ycb_video.py / run_linemod.py do: the estimator and, through the
same chain of star-imports as the reference (estimater.py:10-15), every name the drivers use unqualified."""
from Utils import *  # noqa: F401,F403
from datareader import *  # noqa: F401,F403
import itertools  # noqa: F401
from learning.training.predict_score import *  # noqa: F401,F403
from learning.training.predict_pose_refine import *  # noqa: F401,F403
import yaml  # noqa: F401

from foundationpose_b200.estimater import FoundationPose, register_cameras, register_objects, track_cameras, track_objects  # noqa: F401,E402
