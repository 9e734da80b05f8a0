"""The node's pairing of /compact_data messages with IMU messages (lio_measure_replay, csrc/measure.cc) against a plain-Python restatement
of the reference lines: MeasurementManager::ImuHandler (MeasurementManager.cc:110-116), GetMeasurements with enable_imu = true (:54-108,
MeasurementManager.h:79) and the IMU loop of Estimator::ProcessEstimation (Estimator.cc:2682-2736).  The ProcessImu call list (dt, acc, gyr,
stamp) and the message decisions must agree bit for bit.  No GPU needed."""
from collections import deque

import numpy as np
import pytest

from lio_mapping_b200.node import measure_replay


class Restated:
    """The reference's three functions, fed one arrival at a time: push() returns the messages GetMeasurements decides after it, each as
    (arrival index, processed, its ProcessImu calls)."""

    def __init__(self, delay):
        self.delay = delay
        self.imu_buf, self.msg_buf = deque(), deque()
        self.imu_last_time, self.curr_time = -1.0, -1.0   # MeasurementManager.h:105, Estimator::curr_time_
        self.imu_dropped = 0

    def push(self, i, a):
        delay, imu_buf, msg_buf = self.delay, self.imu_buf, self.msg_buf
        if a[0] == "imu":
            if a[1] <= self.imu_last_time:          # :111-114 "imu message in disorder!"
                self.imu_dropped += 1
            else:
                self.imu_last_time = a[1]
                imu_buf.append(a)
        else:
            msg_buf.append((i, a[1]))
        out = []
        while True:
            if not imu_buf or not msg_buf:          # :62-64
                break
            if imu_buf[-1][1] <= msg_buf[0][1] + delay:      # :66-71 wait for imu
                break
            if imu_buf[0][1] >= msg_buf[0][1] + delay:       # :73-78 throw compact_data
                out.append((msg_buf.popleft()[0], 0, []))
                continue
            idx, stamp = msg_buf.popleft()
            imu_measurements = []
            while imu_buf[0][1] < stamp + delay:     # :83-87
                imu_measurements.append(imu_buf.popleft())
            imu_measurements.append(imu_buf[0])      # :90 one message after laser odom msg, not popped
            calls = []
            ax = ay = az = rx = ry = rz = 0.0        # Estimator.cc:2686
            for m in imu_measurements:
                imu_time = m[1]
                laser_odom_time = stamp + delay
                if imu_time <= laser_odom_time:
                    if self.curr_time < 0:
                        self.curr_time = imu_time
                    dt = imu_time - self.curr_time
                    self.curr_time = imu_time
                    ax, ay, az = m[2]
                    rx, ry, rz = m[3]
                    calls.append((dt, ax, ay, az, rx, ry, rz, imu_time))
                else:
                    dt_1 = laser_odom_time - self.curr_time
                    dt_2 = imu_time - laser_odom_time
                    self.curr_time = laser_odom_time
                    w1 = dt_2 / (dt_1 + dt_2)
                    w2 = dt_1 / (dt_1 + dt_2)
                    ax = w1 * ax + w2 * m[2][0]
                    ay = w1 * ay + w2 * m[2][1]
                    az = w1 * az + w2 * m[2][2]
                    rx = w1 * rx + w2 * m[3][0]
                    ry = w1 * ry + w2 * m[3][1]
                    rz = w1 * rz + w2 * m[3][2]
                    calls.append((dt_1, ax, ay, az, rx, ry, rz, imu_time))
            out.append((idx, 1, calls))
        return out


def restated(delay, arrivals):
    """The whole sequence: (calls (m, 8), events [(arrival index, processed, first call)], IMU messages dropped)."""
    r = Restated(delay)
    calls, events = [], []
    for i, a in enumerate(arrivals):
        for idx, processed, c in r.push(i, a):
            events.append((idx, processed, len(calls)))
            calls += c
    return np.array(calls, np.float64).reshape(-1, 8), events, r.imu_dropped


def _imu(rng, t):
    return ("imu", float(t), tuple(rng.normal(0, 3, 3).tolist()), tuple(rng.normal(0, 0.5, 3).tolist()))


def _published(n_sweeps, odom_io):
    """Sweep indices the odometry publishes: the first sweep never (PointOdometry.cc:302-310), then the io_ratio gate (:725) on
    frame_count_, which counts the sweeps after the first."""
    return [c for c in range(n_sweeps) if c >= 1 and (odom_io < 2 or c % odom_io == 1)]


def _drive(seed, delay, odom_io=1, n_sweeps=12, rate=200.0, jitter=True, lag=0.0, t0=1.0):
    """IMU at `rate` (optionally jittered off the grid) and the published sweeps of a 10 Hz lidar; a message arrives `lag` seconds after its
    stamp (0: in time order)."""
    rng = np.random.default_rng(seed)
    t_end = t0 + 0.1 * n_sweeps + 0.2
    tt = np.arange(int(t0 * rate) - 4, int(t_end * rate)) / rate
    if jitter:
        tt = tt + rng.uniform(-0.3, 0.3, tt.shape) / rate
    events = [(t, 0, _imu(rng, t)) for t in tt]
    for c in _published(n_sweeps, odom_io):
        s = t0 + 0.1 * c
        events.append((s + lag, 1, ("msg", s)))
    events.sort(key=lambda e: (e[0], e[1]))
    return [e[2] for e in events]


def _same(delay, arrivals):
    got_calls, got_events, got_drop = measure_replay(delay, arrivals)
    ref_calls, ref_events, ref_drop = restated(delay, arrivals)
    assert got_events == ref_events
    assert got_drop == ref_drop
    assert got_calls.shape == ref_calls.shape
    assert np.array_equal(got_calls.view(np.uint64), ref_calls.view(np.uint64))   # bit for bit, -0.0 included
    return ref_calls, ref_events, ref_drop


DELAYS = [0.0, 0.05]


@pytest.mark.parametrize("delay", DELAYS)
def test_messages_before_any_imu_are_dropped(delay):
    rng = np.random.default_rng(1)
    arrivals = [("msg", 1.0), ("msg", 1.1)] + [_imu(rng, 1.2 + delay + k / 200) for k in range(10)] + [("msg", 1.25)]
    arrivals += [_imu(rng, 1.3 + delay + k / 200) for k in range(3)]
    calls, events, _ = _same(delay, arrivals)
    assert [e[:2] for e in events] == [(0, 0), (1, 0), (12, 1)]


@pytest.mark.parametrize("delay", DELAYS)
def test_sweeps_ahead_of_the_imu_wait(delay):
    ordered = _drive(2, delay, lag=0.0)
    ahead = [a for a in ordered if a[0] == "msg"] + [a for a in ordered if a[0] == "imu"]    # every message before any IMU
    c0, e0, _ = _same(delay, ordered)
    early = [a for a in ordered if a[0] == "imu" and a[1] < 1.0 + delay]
    rest = [a for a in ordered if not (a[0] == "imu" and a[1] < 1.0 + delay)]
    waited = early + [a for a in rest if a[0] == "msg"] + [a for a in rest if a[0] == "imu"]   # messages wait for later IMU
    c1, e1, _ = _same(delay, waited)
    assert np.array_equal(c0, c1) and [e[1:] for e in e0] == [e[1:] for e in e1]
    _same(delay, ahead)


@pytest.mark.parametrize("delay", DELAYS)
def test_imu_exactly_at_the_laser_time_is_integrated_twice(delay):
    rng = np.random.default_rng(4)
    stamps = [1.0, 1.1]
    arrivals = [_imu(rng, 0.98), _imu(rng, 0.99)]
    for s in stamps:
        arrivals += [_imu(rng, s + delay - 0.005), ("msg", s), _imu(rng, s + delay), _imu(rng, s + delay + 0.004)]
    arrivals += [_imu(rng, 1.3)]
    calls, events, _ = _same(delay, arrivals)
    assert [e[1] for e in events] == [1, 1]
    first_end = events[1][2]
    at = stamps[0] + delay
    assert calls[first_end - 1][7] == at and calls[first_end - 1][0] > 0     # integrated with its own dt
    assert calls[first_end][7] == at and calls[first_end][0] == 0.0           # and again with dt = 0 by the next message


@pytest.mark.parametrize("delay", DELAYS)
def test_interpolated_sample(delay):
    rng = np.random.default_rng(5)
    arrivals = [_imu(rng, 0.995 + delay), ("msg", 1.0), _imu(rng, 1.0037 + delay)]
    calls, events, _ = _same(delay, arrivals)
    assert events == [(1, 1, 0)] and calls.shape[0] == 2
    laser = 1.0 + delay
    assert calls[-1][7] == arrivals[-1][1] and calls[-1][0] == laser - arrivals[0][1]   # the IMU message's own stamp, dt_1
    w1 = (arrivals[-1][1] - laser) / (calls[-1][0] + (arrivals[-1][1] - laser))
    assert 0 < w1 < 1 and calls[-1][1] != arrivals[-1][2][0]


@pytest.mark.parametrize("delay", DELAYS)
def test_out_of_order_imu_is_dropped_and_counted(delay):
    rng = np.random.default_rng(6)
    arrivals = _drive(7, delay, n_sweeps=6)
    imu_idx = [i for i, a in enumerate(arrivals) if a[0] == "imu"]
    for i in imu_idx[20:60:7]:
        arrivals.insert(i, _imu(rng, arrivals[i - 1][1] if arrivals[i - 1][0] == "imu" else 0.5))   # repeated or older stamps
    _, _, dropped = _same(delay, arrivals)
    assert dropped >= 5


@pytest.mark.parametrize("odom_io", [1, 2, 3])
@pytest.mark.parametrize("delay", DELAYS)
@pytest.mark.parametrize("lag", [0.0, 0.03, 0.25])
def test_odom_io_gated_drives(odom_io, delay, lag):
    arrivals = _drive(10 + odom_io, delay, odom_io=odom_io, n_sweeps=13, lag=lag)
    calls, events, _ = _same(delay, arrivals)
    assert sum(e[1] for e in events) >= len(_published(13, odom_io)) - 2


def test_grid_imu_with_a_stamp_on_every_laser_time():
    """200 Hz IMU on the grid and 10 Hz messages with delay 0: every laser time has a sample stamped exactly at it."""
    arrivals = _drive(20, 0.0, n_sweeps=8, jitter=False)
    calls, events, _ = _same(0.0, arrivals)
    starts = [e[2] for e in events if e[1]][1:]
    assert all(calls[s][0] == 0.0 for s in starts)


def test_zero_step_of_the_preintegration():
    """The pairing hands lio_est_process_imu dt = 0 for a sample integrated twice.  The pre-integration it drives keeps delta_p, delta_v,
    sum_dt, the Jacobian and the covariance bit for bit; delta_q is only re-normalised (IntegrationBase.h:302), a change of at most a few
    ulp that the reference's own dt = 0 call makes as well."""
    from lio_mapping_b200.estimator import Pim
    p = Pim(np.array([0.1, 0.2, 9.8]), np.array([0.01, -0.02, 0.03]), np.zeros(3), np.zeros(3), acc_n=0.2, gyr_n=0.02)
    for k in range(5):
        p.push_back(0.005, np.array([0.1 + k * 0.01, 0.2, 9.8]), np.array([0.01, -0.02, 0.03 + k * 1e-3]))
    before = p.get()
    p.push_back(0.0, np.array([0.14, 0.2, 9.8]), np.array([0.01, -0.02, 0.034]))
    after = p.get()
    for k in ("delta_p", "delta_v", "sum_dt", "jacobian", "covariance"):
        assert np.array_equal(before[k], after[k]), k
    assert np.abs(after["delta_q"] - before["delta_q"]).max() <= 4e-16
