"""
A streaming model of adaptive sampling's stop rule (rt_set_adaptive_sampling, DESIGN.md section 4), one accumulation at a time, in
IEEE double as k_adaptive_update computes it:

    Y = luma(radiance) in float32, y = Y - Y_prev, Q += y^2, m = Y / n, v = max(Q / n - m^2, 0), e = sqrt(v / n) / (1 + m)^2,
    stop iff n >= min_samples and e <= max_error              (NaN never stops)

The model keeps each pixel's state at its own count and nothing per sample, so a 4K frame costs a few frames of memory however
many samples run.  Every update also reports the tile structure of the device-wide compaction that follows it: tile t holds the
active-list entries [1024 t, 1024 t + 1024) in ascending pixel order, and the model counts the survivors of each tile, which is what
the look-back over earlier tiles adds up.
"""
import numpy as np

TILE = 1024          # RT_AD_TILE: list entries per CTA of k_adaptive_update


def luma(r):
    """rt_device.cuh's luma() in float32: (x * 0.299f + y * 0.587f) + z * 0.114f"""
    r = np.asarray(r, np.float32)
    return (r[..., 0] * np.float32(0.299) + r[..., 1] * np.float32(0.587)) + r[..., 2] * np.float32(0.114)


def rule(Y, y_prev, q, n):
    """One update of pixels now at n samples: float32 luma Y, the luma Y_prev of the previous update and the sum Q of the earlier
    squared increments -> (the new Q, v before the clamp, e)."""
    Y = np.asarray(Y, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore"):                 # inf - inf gives NaN, as on the device
        y = Y - np.asarray(y_prev, np.float32).astype(np.float64)
        qn = np.asarray(q, np.float64) + y * y
        m = Y / n
        raw = qn / n - m * m
        v = np.where(raw < 0.0, 0.0, raw)              # the kernel's `if (v < 0.0) v = 0.0;`: NaN stays NaN
        d = 1.0 + m
        return qn, raw, np.sqrt(v / n) / (d * d)


class Update:
    """What one update did: active pixels before and after it, and the survivors of every tile of its compaction."""

    def __init__(self, n, active_before, survivors):
        self.n = n
        self.active_before = active_before
        self.survivors = survivors                      # (tiles,) int64
        self.active_after = int(survivors.sum())

    @property
    def tiles(self):
        return len(self.survivors)

    @property
    def empty(self):
        return int((self.survivors == 0).sum())

    @property
    def full(self):
        """Tiles whose every entry survives (the last tile counts as full when all of its entries survive)."""
        size = np.full(self.tiles, TILE, np.int64)
        if self.tiles:
            size[-1] = self.active_before - TILE * (self.tiles - 1)
        return int((self.survivors == size).sum())

    @property
    def partial(self):
        return self.tiles - self.empty - self.full

    def __repr__(self):
        return "n=%d active %d->%d tiles=%d empty=%d full=%d partial=%d" % (
            self.n, self.active_before, self.active_after, self.tiles, self.empty, self.full, self.partial)


class AdaptiveModel:
    """The stop rule over a stream of accumulations of one (h, w) image (a rank's local rows for a partition).  update(acc) takes
    the accumulated radiance after the next sample, as a context with the feature off holds it."""

    def __init__(self, shape, max_error, min_samples):
        self.max_error = float(np.float32(max_error))    # rt_set_adaptive_sampling takes a float
        self.min_samples = int(min_samples)
        self.n = 0
        self.count = np.zeros(shape, np.uint32)
        self.active = np.ones(shape, bool)
        self.y_prev = np.zeros(shape, np.float32)
        self.q = np.zeros(shape, np.float64)
        self.radiance = np.zeros(tuple(shape) + (3,), np.float32)   # each pixel's radiance at its own count
        self.updates = []

    @property
    def n_active(self):
        return int(self.active.sum())

    def update(self, acc):
        """The accumulation after sample n + 1 ((h, w, 3 or 4) float32) -> this update's Update."""
        acc = np.asarray(acc, np.float32)[..., :3]
        return self.update_luma(luma(acc), acc)

    def update_luma(self, Y, acc=None):
        """As update(), from the luma of the accumulation (and the accumulation, kept at each pixel's count when given)."""
        self.n += 1
        n, act = self.n, self.active
        qn, _, e = rule(Y, self.y_prev, self.q, n)
        stop = (n >= self.min_samples) & (e <= self.max_error)
        keep = act & ~stop
        before = int(act.sum())
        kept = keep.ravel()[np.flatnonzero(act.ravel())].astype(np.int64)     # list order = ascending local pixel index
        survivors = np.add.reduceat(kept, np.arange(0, before, TILE)) if before else np.zeros(0, np.int64)
        self.q = np.where(act, qn, self.q)
        self.y_prev = np.where(act, Y, self.y_prev)
        self.count[act] = n
        if acc is not None:
            self.radiance[act] = acc[act]
        self.active = keep
        u = Update(n, before, survivors.astype(np.int64))
        self.updates.append(u)
        return u
