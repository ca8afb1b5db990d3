"""CPU: the smoothing port (oracle/smooth_port.py) -- the One-Euro filter per track and joint that ``spg_smooth_frames``
is held to: equal to the textbook scalar filter on one joint, less jitter at rest, less lag with a larger ``beta``, the
state of absent and non-finite joints kept, and the slots' claim and eviction order."""
import numpy as np
import pytest

from oracle import smooth_port as sp

BASE = np.array([[20, 10], [18, 8], [22, 8], [15, 9], [25, 9], [10, 25], [30, 25], [8, 45], [32, 45], [6, 60], [34, 60],
                 [14, 60], [26, 60], [13, 80], [27, 80], [12, 100], [28, 100]], np.float64)
ALL = (1 << 17) - 1


class TextbookOneEuro:
    """The scalar One-Euro filter of Casiez, Roussel and Vogel, in the port's operation order."""

    def __init__(self, min_cutoff, beta, d_cutoff):
        self.min_cutoff, self.beta, self.d_cutoff = np.float64(min_cutoff), np.float64(beta), np.float64(d_cutoff)
        self.x = self.dx = self.t = None

    @staticmethod
    def alpha(cutoff, dt):
        return np.float64(1.0) / (np.float64(1.0) + np.float64(1.0) / (sp.TWO_PI * cutoff * dt))

    def __call__(self, t, x):
        t, x = np.float64(t), np.float64(x)
        if self.x is None:
            self.x, self.dx, self.t = x, np.float64(0.0), t
            return x
        dt = t - self.t
        dx = (x - self.x) / dt
        ad = self.alpha(self.d_cutoff, dt)
        self.dx = ad * dx + (np.float64(1.0) - ad) * self.dx
        a = self.alpha(self.min_cutoff + self.beta * abs(self.dx), dt)
        self.x, self.t = a * x + (np.float64(1.0) - a) * self.x, t
        return self.x


def _one_joint(x, y):
    xy = np.zeros((1, 17, 2))
    xy[0, 5] = (x, y)
    return xy


@pytest.mark.parametrize("params", [(1.0, 1.0, 1.0), (0.3, 0.007, 1.0), (2.5, 40.0, 0.5)])
def test_one_joint_with_constant_y_is_the_textbook_filter(params):
    rng = np.random.default_rng(7)
    s, ref = sp.Smoother(1, *params), TextbookOneEuro(*params)
    t = 0.0
    for k in range(200):
        t += float(rng.uniform(0.005, 0.1))
        x = 300.0 + 40.0 * np.sin(k / 9.0) + rng.normal(0, 2.0)
        got = s.step(0, t, _one_joint(x, 77.25), [1 << 5], [3])
        want = ref(t, x)
        assert got[0, 5, 0].tobytes() == np.float64(want).tobytes(), k
        assert abs(got[0, 5, 1] - 77.25) <= 2 * np.spacing(77.25)  # a * y + (1 - a) * y rounds


def _person(rng, centre, jitter):
    return BASE * 3.0 + centre + rng.uniform(-jitter, jitter, BASE.shape)


def test_a_still_person_jitters_less():
    rng = np.random.default_rng(11)
    s = sp.Smoother(1)
    raw, out = [], []
    for k in range(90):
        xy = _person(rng, (400.0, 200.0), 1.0)[None]
        raw.append(xy[0])
        out.append(s.step(0, k / 30.0, xy, [ALL], [0])[0])
    raw_motion = np.abs(np.diff(raw[30:], axis=0)).mean()
    smooth_motion = np.abs(np.diff(out[30:], axis=0)).mean()
    assert raw_motion > 0.5 and smooth_motion < 0.3 * raw_motion, (raw_motion, smooth_motion)


def test_lag_falls_as_beta_grows():
    lags = []
    for beta in (0.0, 0.2, 1.0, 5.0):
        s = sp.Smoother(1, min_cutoff=1.0, beta=beta)
        for k in range(60):
            xy = (BASE * 3.0 + (400.0 + 300.0 * k / 30.0, 200.0))[None]  # 300 px/s to the right
            out = s.step(0, k / 30.0, xy, [ALL], [0])
        lags.append(float((xy[0, :, 0] - out[0, :, 0]).mean()))
    assert all(a > b > 0 for a, b in zip(lags, lags[1:])), lags


def test_absent_and_nonfinite_joints_keep_their_state_and_return_with_their_own_dt():
    rng = np.random.default_rng(3)
    s, ref = sp.Smoother(1), sp.Smoother(1)
    frames = [_person(rng, (100.0, 100.0), 2.0)[None] for _ in range(3)]
    s.step(0, 0.0, frames[0], [ALL], [9])
    ref.step(0, 0.0, frames[0], [ALL], [9])
    before = s.slots[0][0].joint.copy()
    xy = frames[1].copy()
    xy[0, 4, 1] = np.nan
    xy[0, 6, 0] = np.inf
    out = s.step(0, 0.05, xy, [ALL & ~(1 << 3)], [9])
    for g in (3, 4, 6):  # passed through raw, state untouched
        assert np.array_equal(out[0, g], xy[0, g], equal_nan=True)
        assert np.array_equal(s.slots[0][0].joint[g], before[g])
    assert s.slots[0][0].joint[0, 4] == 0.05 and s.slots[0][0].mask == ALL
    got = s.step(0, 0.1, frames[2], [ALL], [9])
    want = ref.step(0, 0.1, frames[2], [ALL], [9])  # joints 3, 4, 6 see dt = 0.1, as if frame 1 was not there
    for g in (3, 4, 6):
        assert got[0, g].tobytes() == want[0, g].tobytes(), g
    assert not np.array_equal(got[0, 0], want[0, 0])


def test_a_non_positive_dt_restarts_the_joint():
    s = sp.Smoother(1)
    s.step(0, 1.0, _one_joint(10.0, 10.0), [1 << 5], [0])
    s.step(0, 1.1, _one_joint(12.0, 10.0), [1 << 5], [0])
    out = s.step(0, 1.1, _one_joint(30.0, 11.0), [1 << 5], [0])
    assert tuple(out[0, 5]) == (30.0, 11.0) and tuple(s.slots[0][0].joint[5]) == (30.0, 11.0, 0.0, 0.0, 1.1)


def _ids_in_slots(s):
    return [None if sl is None else sl.id for sl in s.slots[0]]


def test_claims_and_eviction_past_128_ids():
    s = sp.Smoother(1)
    xy = lambda n: np.repeat((BASE + 50.0)[None], n, axis=0)  # noqa: E731
    s.step(0, 0.0, xy(128), [ALL] * 128, list(range(128)))
    assert _ids_in_slots(s) == list(range(128))
    s.step(0, 0.1, xy(64), [ALL] * 64, list(range(64)))                  # slots 0..63 used at clock 2
    s.step(0, 0.2, xy(64), [ALL] * 64, list(range(200, 264)))            # evicts slots 64..127 (last 1), in order
    assert _ids_in_slots(s) == list(range(64)) + list(range(200, 264))
    assert [sl.last for sl in s.slots[0]] == [2] * 64 + [3] * 64 and s.clock[0] == 3
    # ties on last go to the lowest index; a slot this frame used is never evicted
    s.step(0, 0.3, xy(3), [ALL] * 3, [0, 300, 301])
    assert _ids_in_slots(s)[:3] == [0, 300, 301] and s.slots[0][1].mask == ALL
    assert sp.Smoother(1).step(0, 0.0, xy(2), [ALL] * 2, [-1, -1]).tobytes() == xy(2).tobytes()


def test_repeated_ids_and_more_than_128_ids_pass_through_raw():
    s = sp.Smoother(1)
    xy = np.repeat((BASE + 50.0)[None], 130, axis=0)
    xy[1:] += np.arange(1, 130)[:, None, None]
    s.step(0, 0.0, xy, [ALL] * 130, list(range(130)))
    out = s.step(0, 0.1, xy + 5.0, [ALL] * 130, list(range(130)))
    assert _ids_in_slots(s) == list(range(128))  # rows 128 and 129 found no slot this frame used
    assert np.array_equal(out[128:], xy[128:] + 5.0) and not np.array_equal(out[:128], xy[:128] + 5.0)
    s = sp.Smoother(1)
    out = s.step(0, 0.0, xy[:3], [ALL] * 3, [4, 4, 4])
    out = s.step(0, 0.1, xy[:3] + 5.0, [ALL] * 3, [4, 7, 4])
    assert _ids_in_slots(s)[:3] == [4, 7, None]
    assert np.array_equal(out[2], xy[2] + 5.0) and not np.array_equal(out[0], xy[0] + 5.0)
