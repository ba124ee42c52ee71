"""Estimator maps for their tests (test_estimator_maps_host.py, test_gpu_estimator_maps.py): oracle/refs.py's KalmanFilterRef told where
the ground is, as hunter_b200.h's "estimator maps" documents it.

Before each update the height rows' measurement is the map's height under each foot at the predicted state. The prediction does not move
the feet, so that is the previous estimate's foot xy. The lookup is height_map_ref.h (episode_ref.terrain_height, whose Python products
round on their own as the device lookup's do). The filter's own heights are not read on a map and are left as they were."""
import numpy as np

from oracle import refs as R
from height_map_ref import h


def foot_xy(x):
    """The four (x, y) the filter state x looks its feet heights up at."""
    return [(float(x[6 + 3 * c]), float(x[7 + 3 * c])) for c in range(4)]


class MappedKalmanFilterRef(R.KalmanFilterRef):
    """KalmanFilterRef on the estimator map m (an HbTerrain; None: the filter itself). lookups: every (x, y) looked up, in order."""

    def __init__(self, m=None):
        super().__init__()
        self.m = m
        self.lookups = []

    def update(self, dt, quat, wl, al, jpos, jvel, contact, kin, prm=R.KF_PARAMS):
        if self.m is None:
            return super().update(dt, quat, wl, al, jpos, jvel, contact, kin, prm=prm)
        own = self.heights
        pts = foot_xy(self.x)
        self.lookups += pts
        self.heights = np.array([h(self.m, px, py) for px, py in pts])
        try:
            return super().update(dt, quat, wl, al, jpos, jvel, contact, kin, prm=prm)
        finally:
            self.heights = own
