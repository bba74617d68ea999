"""What the reference's cosine (embedder.ts:168-184) gives when one side sits at the ends of the float64 range.

cosineSimilarity computes dot / (sqrt(normA) * sqrt(normB)) in binary64.  With an ordinary partner vector of the same
length, the class of the other vector decides what kind of number comes out.  Each entry: (name, how the vector is
made from a standard-normal one, what the reference returns).  The kinds:

- "finite": an ordinary cosine in [-1, 1];
- "inf":    normA or normB underflows to 0 while the dot does not, so x / 0 = +-Infinity (NaN when the dot is 0 too);
- "zero":   normA or normB overflows to Infinity while the dot stays finite, so x / Infinity = +-0;
- "nan":    NaN for every partner (a zero vector, or a non-finite element).

tests/test_float_range_host.py checks the table against the C oracle and oracle/pyref.py; the GPU suite
(tests/test_gpu_float_range.py) builds its corpora and queries from it.  Powers of two scale exactly, so a class's
vectors keep the direction of the standard-normal vector they come from.
"""
import numpy as np

# exponent -> class.  The boundaries: bf16 / float32 normals start at 2^-126 and bf16 subnormals end at 2^-133; float32
# and bf16 end at 2^128; squares of float64 values underflow below about 2^-537 and overflow above 2^512.
SCALES = {
    -1074: "zero_norm",     # only the elements that are exactly +-2^-1074 survive; their squares underflow
    -565: "inf",
    -160: "finite",
    -149: "finite",
    -140: "finite",         # rounds to bf16 zeros
    -134: "finite",
    -133: "finite",
    -127: "finite",
    -126: "finite",
    -100: "finite",
    -60: "finite",
    0: "finite",
    60: "finite",
    100: "finite",
    127: "finite",
    128: "finite",          # past float32 and bf16
    130: "finite",
    600: "zero",
    1000: "zero",
}

# the kind each class gives against an ordinary partner ("zero_norm": a 2^-1074 vector keeps a few +-2^-1074 elements,
# whose dot with an ordinary partner is nonzero, so its cosine is +-Infinity like the "inf" class)
KIND = {"finite": "finite", "inf": "inf", "zero_norm": "inf", "zero": "zero", "nan": "nan"}

SPECIAL = {
    "all_zero": "nan",
    "one_nan": "nan",
    "one_inf": "nan",
}


def scaled(v, e):
    """v * 2^e, exact as long as the result stays in float64's normal range (np.ldexp rounds only on underflow)."""
    return np.ldexp(np.asarray(v, dtype=np.float64), e)


def special(v, name):
    v = np.array(v, dtype=np.float64)
    if name == "all_zero":
        v[:] = 0.0
    elif name == "one_nan":
        v[len(v) // 2] = np.nan
    elif name == "one_inf":
        v[len(v) // 3] = np.inf
    return v


def matches(kind, score):
    """Does `score` (the cosine against an ordinary partner) belong to `kind`?"""
    if kind == "finite":
        return np.isfinite(score) and -1.0 <= score <= 1.0
    if kind == "inf":
        return np.isinf(score) or np.isnan(score)        # NaN only where the dot is exactly 0
    if kind == "zero":
        return score == 0.0 or np.isnan(score)           # NaN only where the dot overflows
    return np.isnan(score)
