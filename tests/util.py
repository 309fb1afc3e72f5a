"""Shared helpers for the tests: deterministic synthetic corpora, digests of the reference's outputs."""
import hashlib
import json
import os

import numpy as np


def zipf_corpus(path, n_tokens, vocab, seed=0, newline_every=0, tail=True, exponent=1.0):
    """Space-separated tokens w<r> with p(r) ~ 1/r^exponent; optional newline every k tokens
    (k may produce empty lines when 1); optional coverage tail so every id occurs once."""
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, vocab + 1) ** exponent
    p /= p.sum()
    ids = rng.choice(vocab, size=n_tokens, p=p)
    if tail:
        ids = np.concatenate([ids, rng.permutation(vocab)])
    parts = []
    for i, t in enumerate(ids):
        parts.append("w%d" % (t + 1))
        if newline_every and (i + 1) % newline_every == 0:
            parts.append("\n")
            if rng.random() < 0.2:
                parts.append("\n")  # empty sentence
        else:
            parts.append(" ")
    with open(path, "w") as f:
        f.write("".join(parts))
    return path


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def digest(x):
    """SHA-256 of an array's bytes (dtype and shape included) or of a list of words."""
    h = hashlib.sha256()
    if isinstance(x, list):
        h.update(json.dumps(x).encode())
    else:
        a = np.ascontiguousarray(x)
        h.update(("%s %s " % (a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def reference_outputs(section):
    """What the unmodified reference computed for a test (tests/golden/make_reference_outputs.py)."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_outputs.json")) as f:
        return json.load(f)[section]


def planted_topic_corpus(path, vocab=5000, topics=25, sentences=60000, length=20, p_topic=0.5, seed=7):
    """SURVEY Appendix B quality corpus: Zipf words, word r belongs to topic r mod `topics`; every
    sentence has a topic, each token comes from that topic with p_topic, else from the global Zipf."""
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, vocab + 1)
    cdf = np.cumsum(p) / p.sum()
    n = sentences * length
    glob = np.searchsorted(cdf, rng.random(n)) + 1                      # ranks 1..V
    # topic draws: Zipf over the words of the topic = ranks t, t+topics, t+2*topics, ...
    per = vocab // topics
    pt = 1.0 / (np.arange(per) * topics + 1.0)
    cdft = np.cumsum(pt) / pt.sum()
    topic = np.repeat(rng.integers(0, topics, sentences), length)
    k = np.searchsorted(cdft, rng.random(n))
    k = np.minimum(k, per - 1)
    tw = k * topics + topic + 1
    tw = np.where(tw > vocab, glob, tw)
    ids = np.where(rng.random(n) < p_topic, tw, glob).reshape(sentences, length)
    with open(path, "w") as f:
        for row in ids:
            f.write(" ".join("w%d" % r for r in row))
            f.write("\n")
    return path


def topic_purity(words, vectors, topics, top_words=1000, k=10):
    """Mean fraction of the k nearest neighbours (cosine) that share the query word's topic, over the
    `top_words` most frequent words (vocabulary order = frequency order; index 0 is </s>)."""
    v = np.asarray(vectors, np.float64)
    ranks = np.array([int(w[1:]) if w.startswith("w") and w[1:].isdigit() else -1 for w in words])
    ok = ranks >= 0
    v = v / (np.linalg.norm(v, axis=1, keepdims=True) + 1e-12)
    q = np.nonzero(ok)[0][:top_words]
    sims = v[q] @ v.T
    sims[np.arange(len(q)), q] = -np.inf
    sims[:, ~ok] = -np.inf
    nn = np.argpartition(-sims, k, axis=1)[:, :k]
    same = (ranks[nn] % topics) == (ranks[q] % topics)[:, None]
    return float(same.mean())
