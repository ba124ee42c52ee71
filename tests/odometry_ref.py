"""numpy restatement of the odometry of the estimated episodes (hb_rollout_set_odometry, hunter_b200.h "odometry"): the simulated tracking
camera of each robot and the filter's fusion of its messages (KalmanFilterEstimate::updateFromTopic). Shared by test_odometry_host.py and
test_gpu_rollout_odometry.py."""
import numpy as np

from estimation_ref import block_normals

HB_ODOM_MAX_DELAY = 15
HISTORY = HB_ODOM_MAX_DELAY + 1
BLOCK_DRIFT, BLOCK_POSITION = 9, 10            # after the sensors' blocks 0-8 (hb_rollout.cuh)


def normals(seed, block, tick, stream):
    """The 3 normals a camera channel adds sigma times to its 3 values."""
    return np.array(block_normals(int(seed), block, int(tick), int(stream))[:3])     # Python ints: the words must not wrap in int64


class CameraRef:
    """The cameras of B instances: settings[i] (an HbOdometrySetting) for i < len(settings), none beyond. State as the context keeps it
    (history by tick modulo HISTORY, bias), cleared at construction as hb_rollout_set_odometry clears it."""

    def __init__(self, settings, B):
        self.s = [settings[i] if i < len(settings) else None for i in range(B)]
        self.hist = np.zeros((B, HISTORY, 3))
        self.bias = np.zeros((B, 3))

    def due(self, i, tick):
        s = self.s[i]
        return s is not None and s.period_ticks > 0 and tick % s.period_ticks == 0 and tick >= s.delay_ticks

    def read(self, rbd, tick, seed, streams):
        """The read at absolute tick `tick` from the true states rbd (B x 32): (pos (B x 3), has_msg (B,)), state advanced."""
        B = rbd.shape[0]
        pos, has = np.zeros((B, 3)), np.zeros(B, dtype=np.uint8)
        for i in range(B):
            s = self.s[i]
            if s is None or s.period_ticks == 0:
                continue
            if tick == 0:
                self.hist[i] = 0.0; self.bias[i] = 0.0
            self.hist[i, tick % HISTORY] = rbd[i, 3:6]
            if not self.due(i, tick):
                continue
            if s.sigma_drift > 0:
                self.bias[i] = self.bias[i] + s.sigma_drift * normals(seed, BLOCK_DRIFT, tick, streams[i])
            p = self.hist[i, (tick - s.delay_ticks) % HISTORY] + self.bias[i]
            if s.sigma_position > 0:
                p = p + s.sigma_position * normals(seed, BLOCK_POSITION, tick, streams[i])
            pos[i], has[i] = p, 1
        return pos, has


def contact_positions_at(oracle, pos, rbd):
    """Pinocchio's contact positions (12,) with the base at pos and the angles and joints of the estimated rbd (the oracle's kinematics)."""
    q = np.zeros(16)
    q[0:3] = pos; q[3:6] = rbd[0:3]; q[6:16] = rbd[6:16]
    return oracle.rbd(q, np.zeros(16))["cpos"]


def update_from_topic(x_hat, feet_heights, rbd, pos, contact, foot_radius, fk):
    """KalmanFilterEstimate::updateFromTopic of one instance with the camera at the base origin, then updateLinear's position: returns
    (x_hat, feet_heights, rbd) after the message pos. fk (12,): the contact positions with the base at pos (contact_positions_at)."""
    x, h, r = np.array(x_hat, dtype=float), np.array(feet_heights, dtype=float), np.array(rbd, dtype=float)
    x[0:3] = pos
    for c in range(4):
        x[6 + 3 * c:9 + 3 * c] = fk[3 * c:3 * c + 3]
        x[8 + 3 * c] -= foot_radius
        if contact[c]:
            h[c] = x[8 + 3 * c]
    r[3:6] = pos
    return x, h, r
