"""Clock drift control on the host (DESIGN.md §4l, DECIDE D4): map the output card's queued samples to a ppm trim for the drift stage.

The input card paces the audio loop and the output card drains what the loop writes.  When their clocks differ by d ppm, the output
card's queue grows or shrinks by rate * d * 1e-6 samples a second; the drift stage (csrc/drift.cu) makes the played stream run
(1 + ppm 1e-6) times as long, so the queue holds still when ppm = d.  `DriftController` finds that ppm from the queue alone:

* warm-up: the first `warmup` readings are ignored (the card's buffers fill), and the set-point is the median of the next `learn`;
* then a proportional-integral law on the error e = smoothed fill - set-point (samples), with the smoothing an exponential average of
  `smooth_s` seconds that takes the edge off a fill read in steps of a driver period:
      ppm = -(kp e + ki sum(e)),  kp = 2 / (G tau),  ki = 1 / (G tau^2)
  where G = chunk 1e-6 is how many samples one chunk at 1 ppm adds and tau the loop's time constant in chunks (`time_constant_s`):
  a critically damped loop for a queue that integrates the ppm error;
* the result is clamped to +-max_ppm and moves by at most `slew_ppm` per chunk, so the pitch never audibly steps (1000 ppm is 1.7
  cents); the integral stops growing while the output is clamped.

Any constant offset in the readings cancels against the learned set-point, so the free space of the output buffer, negated, serves as
well as its fill.  The state is a small dict (`state()` / `DriftController.from_state`) that a pipeline snapshot carries."""
import math
from typing import Any, Dict, Optional


class DriftController(object):
    """ppm trim of a drift stage from the output card's backlog, read once per chunk after the chunk is written."""

    PARAMS = ('rate', 'chunk', 'max_ppm', 'slew_ppm', 'warmup', 'learn', 'time_constant_s', 'smooth_s')

    def __init__(self, rate: int, chunk: int, max_ppm: float = 500.0, slew_ppm: float = 2.0, warmup: int = 10, learn: int = 20,
                 time_constant_s: float = 60.0, smooth_s: float = 4.0):
        if not (rate > 0 and chunk > 0):
            raise ValueError('the drift controller needs a positive rate and chunk')
        if not (math.isfinite(max_ppm) and 0 < max_ppm <= 2000):
            raise ValueError('the drift controller max_ppm must be within (0, 2000]')
        if not (math.isfinite(slew_ppm) and slew_ppm > 0 and time_constant_s > 0 and smooth_s > 0 and warmup >= 0 and learn >= 1):
            raise ValueError('bad drift controller parameters')
        self.rate, self.chunk = int(rate), int(chunk)
        self.max_ppm, self.slew_ppm = float(max_ppm), float(slew_ppm)
        self.warmup, self.learn = int(warmup), int(learn)
        self.time_constant_s, self.smooth_s = float(time_constant_s), float(smooth_s)
        period = self.chunk / self.rate                     # seconds per chunk
        tau = self.time_constant_s / period                 # chunks
        gain = self.chunk * 1e-6                            # samples the queue gains per chunk at 1 ppm
        self.kp, self.ki = 2.0 / (gain * tau), 1.0 / (gain * tau * tau)
        self.alpha = -math.expm1(-period / self.smooth_s)
        self.seen = 0
        self.readings = []                                  # the readings the set-point is learned from
        self.setpoint: Optional[float] = None
        self.level: Optional[float] = None
        self.integral = 0.0
        self.ppm = 0.0

    def update(self, backlog: float) -> float:
        """One reading of the output card's backlog in samples, taken after the chunk's write; returns the ppm for the next chunk."""
        backlog = float(backlog)
        self.seen += 1
        if self.setpoint is None:
            if self.seen > self.warmup:
                self.readings.append(backlog)
                if len(self.readings) >= self.learn:
                    r = sorted(self.readings)
                    h = len(r) // 2
                    self.setpoint = r[h] if len(r) % 2 else 0.5 * (r[h - 1] + r[h])
                    self.level = self.setpoint
                    self.readings = []
            return self.ppm
        self.level += self.alpha * (backlog - self.level)
        e = self.level - self.setpoint
        want = -(self.kp * e + self.ki * (self.integral + e))
        if abs(want) < self.max_ppm:                        # no wind-up while the output is clamped
            self.integral += e
        want = min(max(want, -self.max_ppm), self.max_ppm)
        self.ppm = min(max(want, self.ppm - self.slew_ppm), self.ppm + self.slew_ppm)
        return self.ppm

    def state(self) -> Dict[str, Any]:
        """The parameters and the state, as plain JSON values."""
        d = {k: getattr(self, k) for k in self.PARAMS}
        d.update(seen=self.seen, readings=list(self.readings), setpoint=self.setpoint, level=self.level, integral=self.integral,
                 ppm=self.ppm)
        return d

    @classmethod
    def from_state(cls, d: Dict[str, Any]) -> 'DriftController':
        """The controller `state()` described, continuing where it was."""
        self = cls(**{k: d[k] for k in cls.PARAMS})
        self.seen, self.readings = int(d['seen']), [float(v) for v in d['readings']]
        self.setpoint = None if d['setpoint'] is None else float(d['setpoint'])
        self.level = None if d['level'] is None else float(d['level'])
        self.integral, self.ppm = float(d['integral']), float(d['ppm'])
        return self
