"""NumPy reference of the fp32 sparse engine's semantics (engine.cu / sparse_kernels.cuh / sparse_v2.cuh).

State: ``{id: (w, state)}`` per table; ``state`` is laid out as ``CudaEngine.gather_rows`` returns it,
``[slot0[dim] | slot1[dim] | scalars]``. One step of a table:
  * the gradients of every valid lookup (every rank, every feature that reads the table) are summed per id and
    counted;
  * the optimizer is applied to the touched rows only, lazily: a row keeps its own step count (Adam's beta powers
    are per row), untouched rows stay as they are;
  * an id is invalid when it is >= vocab (array table) or has bit 63 set (hash table; -1 included): it pulls zeros
    and is never pushed.

Two forms of the optimizer step:
  ``exact=True``   float32 replicas of exb_math.h's operation order for `default`, `sgd` and `test` (plus the per-row
                   beta powers of Adam / Adamax). With power-of-two learning rates and momenta and dyadic gradients
                   (small integers x 2^-6, whose sums are exact in fp32 in any order) every product is exact, so each
                   result is one correctly rounded operation: FMA contraction and the order of the atomics cannot
                   change it, and the device must match bit for bit.
  ``exact=False``  float64 Keras formulas for every optimizer, applied lazily per row, plus a per-element error bound
                   for an fp32 implementation that uses sqrt.approx / __fdividef (see ``bound``).
"""
import numpy as np

from openembedding_b200.config import normalize_optimizer, optimizer_slot_inits

F32 = np.float32
U32 = 2.0 ** -24          # unit roundoff of fp32
BOUND_C = 8.0             # the one constant of the error bound: C * u * sum_t t * kappa_t * |terms of step t|
EXACT_CATEGORIES = ("default", "sgd", "test")


def hash64(x):
    """exb_hash64 (splitmix64 finaliser): home slot of a key in a hash shard is hash64(key) & (capacity - 1)"""
    m = (1 << 64) - 1
    x &= m
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & m
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & m
    x ^= x >> 31
    return x


def valid_ids(ids, vocab, is_hash):
    """mask of the ids the engine looks up / updates (int64 ids; bit 63 set == negative)"""
    ids = np.asarray(ids, dtype=np.int64)
    if is_hash:
        return ids >= 0
    return (ids >= 0) & (ids < vocab)


def dyadic(rng, shape, k=64, shift=6):
    """non-zero integers in [-k, k] x 2^-shift: any sum of a few thousand of them is exact in fp32"""
    v = rng.integers(1, k + 1, size=shape) * rng.choice([-1, 1], size=shape)
    return (v * 2.0 ** -shift).astype(F32)


def f32_config(cfg):
    """the optimizer config with every hyper-parameter rounded to fp32, as the device uses them"""
    c = normalize_optimizer(cfg)
    return {k: (float(F32(v)) if isinstance(v, float) else v) for k, v in c.items()}


def _slots(cat):
    return {"default": 0, "adadelta": 2, "adagrad": 1, "adam": 2, "adamax": 2, "ftrl": 2, "rmsprop": 2,
            "sgd": 1, "test": 0}[cat]


def _nscalars(cat):
    return {"adam": 2, "adamax": 1, "test": 2}.get(cat, 0)


# ------------------------------------------------------------------ float32 replicas (exb_math.h operation order)
def scalars_f32(c, sc, cnt):
    """per-row prologue on the trailing scalars (opt_row_prologue): returns (new scalars, rc.a, rc.b)"""
    cat = c["category"]
    sc = sc.astype(F32).copy()
    a = b = None
    if cat == "adam":
        sc[:, 0] = sc[:, 0] * F32(c["beta_1"])
        sc[:, 1] = sc[:, 1] * F32(c["beta_2"])
    elif cat == "adamax":
        sc[:, 0] = sc[:, 0] * F32(c["beta_1"])
    elif cat == "test":
        a = F32(c["flip"]) - sc[:, 0]
        sc[:, 0] = a
        b = np.maximum(cnt, 1).astype(F32)
    return sc, a, b


def step_f32(c, w, s, g, cnt):
    """one update of rows w [n, dim], state s [n, sd] with summed gradients g and counts cnt, in fp32 (exact
    categories; Adam / Adamax: the scalars only)"""
    cat, dim = c["category"], w.shape[1]
    w, s = w.astype(F32).copy(), s.astype(F32).copy()
    ns = _slots(cat) * dim
    sc, a, b = scalars_f32(c, s[:, ns:], cnt)
    s[:, ns:] = sc
    with np.errstate(all="ignore"):
        if cat == "default":
            lr = F32(c["learning_rate"])
            if lr != 0:
                w = w - lr * g
        elif cat == "sgd":
            lr, mom = F32(c["learning_rate"]), F32(c["momentum"])
            s0 = s[:, :dim] * mom + lr * g
            s[:, :dim] = s0
            w = w - (s0 * mom + lr * g) if c["nesterov"] else w - s0
        elif cat == "test":
            lr = F32(c["learning_rate"])
            w = w + ((lr * g) / b[:, None] + a[:, None])
        elif cat not in ("adam", "adamax"):
            raise ValueError("no float32 replica of " + cat)
    return w, s


# ------------------------------------------------------------------ float64 Keras formulas + error terms
def step_f64(c, w, s, g, t):
    """one lazy Keras step in fp64 of rows w [n, dim] with state s [n, sd] (device layout; sgd keeps the
    velocity with the device's sign) and per-row step numbers t [n] (1 for a row's first update).
    Returns (w, s, wterm, sterm): wterm / sterm are, per element, the magnitudes an fp32 evaluation of this step
    rounds (|inputs| + |increments|), already weighted by the conditioning of the step (kappa)."""
    cat, dim = c["category"], w.shape[1]
    w, s = w.astype(np.float64).copy(), s.astype(np.float64).copy()
    w0 = w.copy()
    lr = c["learning_rate"]
    s0, s1 = s[:, :dim], s[:, dim:2 * dim]
    st0, st1 = np.zeros_like(w), np.zeros_like(w)
    kappa = np.ones((w.shape[0], 1))
    tt = t.astype(np.float64)[:, None]
    wextra = np.zeros_like(w)
    if cat == "default":
        w = w - lr * g
    elif cat == "sgd":
        mom = c["momentum"]
        st0 = np.abs(s0 * mom) + np.abs(lr * g)
        s0[:] = s0 * mom + lr * g
        w = w - (s0 * mom + lr * g) if c["nesterov"] else w - s0
    elif cat == "adagrad":
        st0 = np.abs(s0) + g * g
        s0[:] = s0 + g * g
        w = w - lr * g / (np.sqrt(s0) + c["epsilon"])
    elif cat == "adadelta":
        rho, eps = c["rho"], c["epsilon"]
        st0 = np.abs(s0 * rho) + (1 - rho) * g * g
        s0[:] = s0 * rho + (1 - rho) * g * g
        upd = g * np.sqrt(s1 + eps) / np.sqrt(s0 + eps)
        st1 = np.abs(s1 * rho) + (1 - rho) * upd * upd
        s1[:] = s1 * rho + (1 - rho) * upd * upd
        w = w - lr * upd
    elif cat == "adam":
        b1, b2, eps = c["beta_1"], c["beta_2"], c["epsilon"]
        st0 = np.abs(s0 * b1) + (1 - b1) * np.abs(g)
        st1 = np.abs(s1 * b2) + (1 - b2) * g * g
        s0[:] = s0 * b1 + (1 - b1) * g
        s1[:] = s1 * b2 + (1 - b2) * g * g
        p1, p2 = b1 ** tt, b2 ** tt
        s[:, 2 * dim:2 * dim + 2] = np.concatenate([p1, p2], 1)
        lr_t = lr * np.sqrt(1 - p2) / (1 - p1)
        w = w - lr_t * s0 / (np.sqrt(s1) + eps)
        # the fp32 beta powers carry t roundings each: relative error t*u*(p/(1-p)) in 1 - p
        kappa = 1 + tt * (p2 / (2 * (1 - p2)) + p1 / (1 - p1))
    elif cat == "adamax":
        b1, b2, eps = c["beta_1"], c["beta_2"], c["epsilon"]
        st0 = np.abs(s0 * b1) + (1 - b1) * np.abs(g)
        s0[:] = s0 * b1 + (1 - b1) * g
        s1[:] = np.maximum(s1 * b2, np.abs(g))
        st1 = np.abs(s1)
        p1 = b1 ** tt
        s[:, 2 * dim:2 * dim + 1] = p1
        w = w - lr / (1 - p1) * s0 / (s1 + eps)
        kappa = 1 + tt * p1 / (1 - p1)
    elif cat == "rmsprop":
        rho, mom, eps = c["rho"], c["momentum"], c["epsilon"]
        st0 = np.abs(s0 * rho) + (1 - rho) * g * g
        s0[:] = s0 * rho + (1 - rho) * g * g
        inc = lr * g / np.sqrt(s0 + eps)
        st1 = np.abs(s1 * mom) + np.abs(inc)
        s1[:] = s1 * mom + inc
        w = w - s1
    elif cat == "ftrl":
        l1, l2, l2s = c["l1_regularization_strength"], c["l2_regularization_strength"], \
            c["l2_shrinkage_regularization_strength"]
        pw, beta = -c["learning_rate_power"], c["beta"]
        gs = g + 2 * l2s * w
        n_new = s0 + g * g
        sigma = (n_new ** pw - s0 ** pw) / lr
        st0 = np.abs(s0) + g * g
        st1 = np.abs(s1) + np.abs(gs) + np.abs(sigma * w) + (n_new ** pw + s0 ** pw) / lr * np.abs(w)
        s1[:] = s1 + gs - sigma * w
        s0[:] = n_new
        quad = n_new ** pw / lr + 2 * (l2 + beta / (2 * lr))
        w = np.where(np.abs(s1) > l1, (np.sign(s1) * l1 - s1) / quad, 0.0)
        # w is recomputed from z: its error is z's error over the quadratic term
        wextra = (np.abs(s1) + st1) / quad
    elif cat == "test":
        raise ValueError("the test optimizer has an exact replica only")
    wterm = np.abs(w0) + kappa * np.abs(w - w0) + np.abs(lr * g) + wextra
    sterm = np.zeros_like(s)
    sterm[:, :dim] = st0 if _slots(cat) > 0 else 0.0
    if _slots(cat) > 1:
        sterm[:, dim:2 * dim] = st1
    return w, s, tt * wterm, tt * np.abs(sterm) + tt * np.abs(s) * (np.arange(s.shape[1]) >= 2 * dim)


class TableRef:
    """Reference of one table. ``exact``: float32 replica (default / sgd / test; Adam / Adamax scalars); else the
    float64 Keras form, which also accumulates the error bound ``bound(ids)`` of an fp32 implementation."""

    def __init__(self, dim, vocab, is_hash, cfg, init_value=0.0, exact=True):
        self.dim, self.vocab, self.is_hash, self.exact = int(dim), int(vocab), bool(is_hash), exact
        self.c = f32_config(cfg)
        cat = self.c["category"]
        if exact and cat not in EXACT_CATEGORIES + ("adam", "adamax"):
            raise ValueError("no exact replica of " + cat)
        slots, scal = optimizer_slot_inits(self.c)
        self.sd = len(slots) * self.dim + len(scal)
        self.s_init = np.array([v for v in slots for _ in range(self.dim)] + scal, dtype=np.float64)
        self.w_init = np.full(self.dim, F32(init_value), dtype=np.float64)
        self.rows = {}          # id -> [w, s, steps, wbound_terms, sbound_terms]
        self.dt = F32 if exact else np.float64

    # ---- rows
    def _row(self, i):
        r = self.rows.get(i)
        if r is None:
            return [self.w_init.astype(self.dt), self.s_init.astype(self.dt), 0,
                    np.zeros(self.dim), np.zeros(self.sd)]
        return r

    def seed(self, ids, w, s=None):
        """rows written through scatter_rows (state None: the optimizer's initial state)"""
        for k, i in enumerate(np.asarray(ids, dtype=np.int64).tolist()):
            st = self.s_init if s is None else s[k]
            self.rows[i] = [np.asarray(w[k]).astype(self.dt), np.asarray(st).astype(self.dt), 0,
                            np.zeros(self.dim), np.zeros(self.sd)]

    def get(self, ids):
        """(weights [n, dim], state [n, sd]) of ids as gather_rows returns them (missing: initial values)"""
        ids = np.asarray(ids, dtype=np.int64).tolist()
        w = np.zeros((len(ids), self.dim), dtype=self.dt)
        s = np.zeros((len(ids), self.sd), dtype=self.dt)
        for k, i in enumerate(ids):
            r = self._row(i)
            w[k], s[k] = r[0], r[1]
        return w, s

    def pull(self, ids):
        """what a pull returns: the row, zeros for an invalid id"""
        w, _ = self.get(ids)
        w[~valid_ids(ids, self.vocab, self.is_hash)] = 0
        return w

    def bound(self, ids):
        """per-element error bound (weights, state) of an fp32 implementation after the steps so far"""
        ids = np.asarray(ids, dtype=np.int64).tolist()
        wb = np.stack([self._row(i)[3] for i in ids]) * BOUND_C * U32
        sb = np.stack([self._row(i)[4] for i in ids]) * BOUND_C * U32
        return wb, sb

    def materialized(self):
        return set(self.rows)

    # ---- one step
    def reduce(self, ids, grads):
        """sum and count the gradients of the valid lookups: (unique ids, summed grads, counts)"""
        ids = np.asarray(ids, dtype=np.int64).reshape(-1)
        grads = np.asarray(grads).reshape(ids.size, self.dim)
        ok = valid_ids(ids, self.vocab, self.is_hash)
        ids, grads = ids[ok], grads[ok]
        u, inv, cnt = np.unique(ids, return_inverse=True, return_counts=True)
        g = np.zeros((u.size, self.dim), dtype=self.dt)
        np.add.at(g, inv, grads.astype(self.dt))
        return u, g, cnt

    def step(self, ids, grads):
        """ids [n] (the lookups of every rank and feature reading the table), grads [n, dim]; returns the unique
        valid ids that were updated"""
        u, g, cnt = self.reduce(ids, grads)
        if u.size == 0:
            return u
        rows = [self._row(i) for i in u.tolist()]
        w = np.stack([r[0] for r in rows])
        s = np.stack([r[1] for r in rows])
        if self.exact:
            w, s = step_f32(self.c, w, s, g, cnt)
            for k, i in enumerate(u.tolist()):
                self.rows[i] = [w[k], s[k], rows[k][2] + 1, rows[k][3], rows[k][4]]
            return u
        t = np.array([r[2] + 1 for r in rows])
        w, s, wt, stt = step_f64(self.c, w, s, g, t)
        for k, i in enumerate(u.tolist()):
            self.rows[i] = [w[k], s[k], t[k], rows[k][3] + wt[k], rows[k][4] + stt[k]]
        return u
