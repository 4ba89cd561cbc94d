"""Deterministic synthetic inputs for the WaveNet hot path.

Two generators:

* ``GlibcRand`` + ``reference_test_inputs``: a numpy replay of glibc's ``srand``/``rand``
  (TYPE_3 additive feedback generator) and of the input construction in the reference's
  integration test (nv_wavenet_test.cu:36-111, 217-219; Matrix::randomize matrix.cpp:38-56).
  With the same seed it reproduces, bit for bit, the weights / Lh / selectors the reference
  test feeds its CPU and GPU implementations -- tests/test_oracle_pin.py proves that against
  oracle/_ref (the reference's own Matrix::randomize + libc rand()).  This lets the GPU box,
  which has no /root/reference, regenerate the reference's test vectors.

* ``synthetic_inputs``: counter-based (numpy PCG64) inputs with the same distributions
  (U(-0.25/rows, 0.25/rows) style, SURVEY.md §8d) for arbitrary shapes.
"""
import numpy as np


class GlibcRand:
    """glibc random_r TYPE_3 (r[i] = r[i-3] + r[i-31], output >> 1), i.e. what rand() returns
    after srand(seed).  State lives here; the stepping loop runs in oracle/liboracle.so
    (wno_glibc_rand_fill) when available, else in Python."""

    def __init__(self, seed):
        self.srand(seed)

    def srand(self, seed):
        seed = int(seed) & 0xFFFFFFFF
        if seed == 0:
            seed = 1
        st = np.zeros(33, dtype=np.uint32)
        word = seed if seed < (1 << 31) else seed - (1 << 32)     # int32_t word = seed
        st[0] = seed
        for i in range(1, 31):
            hi = int(word / 127773)                               # C division truncates toward zero
            lo = word - hi * 127773
            word = 16807 * lo - 2836 * hi
            if word < 0:
                word += 2147483647
            st[i] = word
        st[31] = 3                                                # fptr = &state[rand_sep]
        st[32] = 0                                                # rptr = &state[0]
        self._st = st
        self.rand_array(310)                                      # srandom_r discards 10*31 outputs

    def rand(self):
        return int(self.rand_array(1)[0])

    def rand_array(self, n):
        """n successive rand() values (int32 array)."""
        out = np.empty(n, dtype=np.int32)
        fill = _c_fill()
        if fill is not None:
            import ctypes as C
            fill(self._st.ctypes.data_as(C.POINTER(C.c_uint32)), n, out.ctypes.data_as(C.POINTER(C.c_int32)))
            return out
        st = [int(x) for x in self._st[:31]]
        f, r = int(self._st[31]), int(self._st[32])
        for i in range(n):
            v = (st[f] + st[r]) & 0xFFFFFFFF
            st[f] = v
            out[i] = v >> 1
            f = f + 1 if f < 30 else 0
            r = r + 1 if r < 30 else 0
        self._st[:31] = st
        self._st[31], self._st[32] = f, r
        return out


_FILL = [False]


def _c_fill():
    if _FILL[0] is False:
        try:
            import ctypes as C
            from oracle.pyoracle import Oracle
            fn = Oracle.lib().wno_glibc_rand_fill
            fn.restype = None
            fn.argtypes = [C.POINTER(C.c_uint32), C.c_long, C.POINTER(C.c_int32)]
            _FILL[0] = fn
        except Exception:
            _FILL[0] = None
    return _FILL[0]


RAND_MAX = 2147483647


def randomize(rng, rows, cols, mean, scale):
    """Matrix::randomize(mean, scale, sparsity=0) on a col-major rows x cols matrix
    (matrix.cpp:38-56).  Returns the col-major flat float32 storage.

    Per element (row-major visiting order): one rand() for the sparsity test, one for the value;
    r = (float)rand() / (float)RAND_MAX; r -= 0.5 (in double, stored to float); r = r*scale + mean.
    """
    n = rows * cols
    raw = rng.rand_array(2 * n)[1::2]
    r = raw.astype(np.float32) / np.float32(RAND_MAX)          # float / float
    r = (r.astype(np.float64) - 0.5).astype(np.float32)         # r -= 0.5 promotes to double
    r = r * np.float32(scale) + np.float32(mean)                # float ops
    r = r.astype(np.float32).reshape(rows, cols)                # visiting order: row outer, col inner
    return np.ascontiguousarray(r.T).reshape(-1)                # col-major storage: data[row + col*rows]


def _create_matrix(rng, r, c):
    """createMatrix (nv_wavenet_test.cu:36-42): scale = 0.5 / rows (computed in double, stored to float)."""
    return randomize(rng, r, c, np.float32(0.0), np.float32(0.5 / r))


def reference_test_inputs(rng, R, S, A, L, B, N):
    """Replays runTest<>() input construction (nv_wavenet_test.cu:44-220) on the given rand stream."""
    f = np.float32
    mean = f(0.0)
    scale = f(0.5 / R)
    rng.rand_array(2 * B)                                        # yInPrev/yInCur draws (:54-57)
    w = {}
    w["selectors"] = randomize(rng, B, N, f(0.5), f(1.0)).reshape(N, B)
    w["embPrev"] = randomize(rng, R, A, mean, scale).reshape(A, R)
    w["embCur"] = randomize(rng, R, A, mean, scale).reshape(A, R)
    keys = ["Wprev", "Wcur", "Bh", "Wres", "Bres", "Wskip", "Bskip"]
    shapes = [(2 * R, R), (2 * R, R), (2 * R, 1), (R, R), (R, 1), (S, R), (S, 1)]
    per = {k: [] for k in keys}
    for _ in range(L):
        for k, (r, c) in zip(keys, shapes):
            per[k].append(_create_matrix(rng, r, c))
        rng.rand_array(2 * S * B)                                # skipOut[l] = createMatrix(S,batch)
    for k in keys:
        w[k] = np.stack(per[k])
    rng.rand_array(2 * R * B * N * (L + 1))                      # Xt[sample][layer] = createMatrix(R,batch)
    w["Wzs"] = randomize(rng, A, S, mean, scale)
    w["Bzs"] = randomize(rng, A, 1, mean, scale)
    w["Wza"] = randomize(rng, A, A, mean, scale)
    w["Bza"] = randomize(rng, A, 1, mean, scale)
    w["Lh"] = randomize(rng, 2 * R, N * L * B, mean, scale).reshape(N, L, B, 2 * R)
    return w


# The reference test's groups: (seed, [(R,S,A,L, impl, ...)...]) -- nv_wavenet_test.cu:343-394.
# Within a group the rand() stream continues from one runTest to the next.
REFERENCE_TEST_GROUPS = [
    (3, [(32, 128, 256, None)] * 4),
    (10, [(64, 128, 256, None)] * 4),
    (30, [(64, 256, 256, None)] * 4),
    (50, [(128, 256, 256, None)] * 2),
    (70, [(64, 128, 512, None), (128, 256, 1024, 12)]),
]


def synthetic_inputs(seed, R, S, A, L, B, N, lh_scale=None, dtype=np.float32):
    """Counter-based inputs with the reference test's distributions (SURVEY.md §8d)."""
    g = np.random.Generator(np.random.PCG64(seed))

    def u(shape, scale):
        return ((g.random(shape, dtype=np.float32) - np.float32(0.5)) * np.float32(scale)).astype(np.float32)

    w = {
        "selectors": g.random((N, B), dtype=np.float32),
        "embPrev": u((A, R), 0.5 / R), "embCur": u((A, R), 0.5 / R),
        "Wprev": u((L, 2 * R * R), 0.5 / (2 * R)), "Wcur": u((L, 2 * R * R), 0.5 / (2 * R)),
        "Bh": u((L, 2 * R), 0.5 / (2 * R)),
        "Wres": u((L, R * R), 0.5 / R), "Bres": u((L, R), 0.5 / R),
        "Wskip": u((L, S * R), 0.5 / S), "Bskip": u((L, S), 0.5 / S),
        "Wzs": u(A * S, 0.5 / R), "Bzs": u(A, 0.5 / R), "Wza": u(A * A, 0.5 / R), "Bza": u(A, 0.5 / R),
        "Lh": u((N, L, B, 2 * R), (0.5 / R) if lh_scale is None else lh_scale),
    }
    return w


def lively_inputs(seed, R, S, A, L, B, N):
    """Like synthetic_inputs but with O(1) weight scales so that gates, logits and the sampled
    distribution are far from uniform (the reference test's 0.5/R scale gives p ~= 1/A)."""
    g = np.random.Generator(np.random.PCG64(seed))

    def n(shape, std):
        return (g.standard_normal(shape, dtype=np.float32) * np.float32(std)).astype(np.float32)

    w = {
        "selectors": g.random((N, B), dtype=np.float32),
        "embPrev": n((A, R), 0.7), "embCur": n((A, R), 0.7),
        "Wprev": n((L, 2 * R * R), 0.7 / np.sqrt(R)), "Wcur": n((L, 2 * R * R), 0.7 / np.sqrt(R)),
        "Bh": n((L, 2 * R), 0.1),
        "Wres": n((L, R * R), 0.5 / np.sqrt(R)), "Bres": n((L, R), 0.05),
        "Wskip": n((L, S * R), 0.5 / np.sqrt(R)), "Bskip": n((L, S), 0.05),
        "Wzs": n(A * S, 1.0 / np.sqrt(S)), "Bzs": n(A, 0.1), "Wza": n(A * A, 2.0 / np.sqrt(A)), "Bza": n(A, 0.1),
        "Lh": n((N, L, B, 2 * R), 0.5),
    }
    return w


def export_inputs(seed, R, S, A, L, B, N, peak=5.0):
    """The configuration a PyTorch model's export_weights() hands NVWaveNet, on lively_inputs weights: run it with
    tanh_embed=False.  embPrev is zero and embCur ~ N(0, 1) (an nn.Embedding, not bounded by the tanh), there are no output
    biases (Bzs = Bza = 0), and the last layer's residual weights and bias are zero (the layer NVWaveNet appends).
    Wza is lively_inputs' times `peak`, so the sampled distribution is peaked as a trained model's is: at L16 R64 S256 A256,
    peak 5 gives a mean max-probability of about 0.46 and a logit spread of about 20 (peak 2.5: 0.16 and 10).  That a trained
    model looks like this is an assumption: no trained checkpoint is part of the project."""
    w = lively_inputs(seed, R, S, A, L, B, N)
    g = np.random.Generator(np.random.PCG64(seed + 0x5EED))
    w["embPrev"] = np.zeros((A, R), np.float32)
    w["embCur"] = g.standard_normal((A, R), dtype=np.float32)
    w["Bzs"] = np.zeros(A, np.float32)
    w["Bza"] = np.zeros(A, np.float32)
    w["Wres"][L - 1] = 0
    w["Bres"][L - 1] = 0
    w["Wza"] = (w["Wza"] * np.float32(peak)).astype(np.float32)
    return w
