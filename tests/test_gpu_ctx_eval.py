"""The evaluator on a training context's own tables (w2b_ctx_compute_accuracy, w2b_ctx_analogy_answers,
w2b_ctx_analogy_topk, w2b_ctx_nearest; Trainer.compute_accuracy and friends).

1. Pinned to the reference through a context: every analogy case and every packed case, uploaded as u (v = -0, which
   leaves every u bit as it is, so export() returns the case's vectors), answers every question as the reference's
   compute_accuracy does on the case's file (stored digests), on the filter and on the SIMT path.
2. Equal to the file round trip where u and v both matter: report text, answers, top-k ids and score bits, nearest
   lists and the route (bit domain or fp32, filter or SIMT) equal the file-based calls on the file written from
   export(), at every width and training bit level, with and without re-quantisation and a threshold.
3. A trained context, after one epoch and after a second one resumed from a checkpoint, gives what its exported file
   gives, and an evaluation changes nothing a later epoch reads.
4. The CLI's per-epoch -eval lines equal compute_accuracy's last two lines on the epoch's vector file.
5. Refused calls leave the context as it was."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import word2bits_b200 as w2b
from word2bits_b200._lib import EINVAL, ESTATE, lib
from tests import analogy_cases as ac
from tests import packed_cases as pc
from tests.util import digest, reference_outputs, zipf_corpus

pytestmark = pytest.mark.gpu
KS = (1, 10, 100, 1024)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN_CLI = os.path.join(ROOT, "word2bits_b200", "word2bits")
ACC_CLI = os.path.join(ROOT, "word2bits_b200", "compute_accuracy")
# widths of the cases w2b_create refuses (layer1_size above 4096, or above 1024 and not a multiple of 4 where the
# register kernel trains): none of the analogy or packed cases' widths (1 ... 2000) is refused
REFUSED_WIDTHS = ()


class _simt:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.old = os.environ.get("W2B_EVAL_SIMT")
        os.environ["W2B_EVAL_SIMT"] = "1" if self.on else "0"

    def __exit__(self, *a):
        if self.old is None:
            del os.environ["W2B_EVAL_SIMT"]
        else:
            os.environ["W2B_EVAL_SIMT"] = self.old


def _context(u, v, bits):
    V, D = u.shape
    t = w2b.Trainer(None, vocab_size=V, size=D, bitlevel=bits, threads=1)
    t.upload_raw(u, v)
    return t


def _as_u(vec):
    """(u, v) whose quantize(u + v) at bit level 0 is vec bit for bit: x + (-0) = x for every x, -0 included."""
    return vec, np.full(vec.shape, -0.0, np.float32)


# ---------------------------------------------------------------------------------------- 1. pinned to the reference
def _pinned(vf, qf, train_bits, eval_bits, th, stored, name):
    names, vec = pc.read_vectors(vf)
    if vec.shape[1] in REFUSED_WIDTHS:
        pytest.skip("w2b_create refuses D = %d" % vec.shape[1])
    t = _context(*_as_u(vec), train_bits)
    try:
        for simt in (False, True):
            with _simt(simt):
                got = t.analogy_answers(qf, names=names, bitlevel=eval_bits, threshold=th)
            assert digest(got) == stored[name]["answers"], "%s simt=%d" % (name, simt)
        with _simt(False):
            text, _ = t.compute_accuracy(qf, names=names, bitlevel=eval_bits, threshold=th)
        assert text == stored[name]["report"]
    finally:
        t.close()


@pytest.mark.parametrize("name", sorted(ac.CASES))
def test_analogy_case_through_a_context_answers_like_the_reference(tmp_path, name):
    vf, qf, b, th = ac.build(name, str(tmp_path))
    _pinned(vf, qf, 0, b, th, reference_outputs("analogy"), name)


@pytest.mark.parametrize("name", sorted(pc.CASES))
def test_packed_case_through_a_context_answers_like_the_reference(tmp_path, name):
    pf, vf, qf, b, th = pc.build(name, str(tmp_path))
    _pinned(vf, qf, b, 0, th, pc.reference_answers(), name)  # trained at the case's level: the bit-domain route


# ------------------------------------------------------------------------------------ 2. equal to the file round trip
REQUANT = {0: 2, 1: 2, 2: 1, 3: 1, 5: 2, 8: 4}


def _crafted(kind, D, bits, seed):
    """(u, v, names, questions): quantize(u + v) differs from quantize(u) on most values; rows with u = -v (exact
    zeros), rows of -0.0 + -0.0, duplicate names.  kind "all_equal": 1500 equal rows (every score ties: the candidate
    lists overflow into the SIMT fall-back); "ties": random rows at D = 8 (1-bit rows tie by the hundred)."""
    rng = np.random.default_rng(seed)
    V = 1500 if kind == "all_equal" else 700
    if kind == "all_equal":
        u = np.tile(rng.normal(size=(1, D)), (V, 1)).astype(np.float32) * 0.4
        v = np.tile(rng.normal(size=(1, D)), (V, 1)).astype(np.float32) * 0.4
    else:
        u = (rng.normal(size=(V, D)) * 0.4).astype(np.float32)
        v = (rng.normal(size=(V, D)) * 0.4).astype(np.float32)
        v[1:40:3] = -u[1:40:3]                                          # u + v = +0 exactly
        u[2:40:3] = -0.0
        v[2:40:3] = -0.0                                                # -0 + -0 = -0
        v[40:60] = np.where(rng.random((20, D)) < 0.5, -u[40:60], v[40:60])  # zeros in some columns
    names = ["w%d" % i for i in range(V)]
    for r in rng.choice(np.arange(100, V), 20, replace=False):
        names[r] = names[rng.integers(1, r)]
    qs = [[names[k] for k in rng.integers(0, min(V, 600), 4)] for _ in range(300)]
    qs += [["missingword", names[1], names[2], names[3]], [names[1]] * 4, [names[1], names[2], names[3], names[3]]]
    return u, v, names, qs


def _files(t, names, bits, d):
    """The files of the context's export(): word2vec-binary, and packed at 1 and 2 bits."""
    vec = t.export()
    vf = os.path.join(d, "vec.bin")
    ac.write_vectors(vf, names, vec)
    pf = None
    if bits in (1, 2):
        pf = os.path.join(d, "vec.packed")
        pc.write_packed(pf, names, pc.pack_rows(vec, bits), vec.shape[1], bits)
    return vf, pf


def _same_lists(a, b, tag):
    assert np.array_equal(a[0], b[0]), tag
    assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)), tag


def _stats(st):
    return {k: v for k, v in st.items() if k != "gpu_ms"}


def _equal_to_round_trip(t, names, bits, qf, wf, d, calls=("acc", "ans", "topk", "near"), thresholds=(0, 500)):
    vf, pf = _files(t, names, bits, d)
    before = t.table_checksum(), t.get_state()
    runs = [(0, 0), (REQUANT[bits], 0)] + [(0, th) for th in thresholds if th]
    for bl, th in runs:
        bit_route = bits in (1, 2) and bl in (0, bits)
        for simt in (False, True):
            tag = "train bits %d, bitlevel %d, threshold %d, simt %d" % (bits, bl, th, simt)
            with _simt(simt):
                if "acc" in calls:
                    text, acc = t.compute_accuracy(qf, names=names, bitlevel=bl, threshold=th)
                    ftext, facc = w2b.compute_accuracy(vf, qf, bitlevel=bl, threshold=th)
                    assert text == ftext, tag
                    keep = ("questions_total", "questions_seen", "correct", "semantic_correct", "semantic_seen",
                            "syntactic_correct", "syntactic_seen", "vocab", "size")
                    assert {k: acc[k] for k in keep} == {k: facc[k] for k in keep}, tag
                    if bit_route:
                        ptext, pacc = w2b.compute_accuracy_packed(pf, qf, threshold=th)
                        assert ptext == text and (pacc["candidates"], pacc["rescored"]) == (acc["candidates"], acc["rescored"]), tag
                    else:
                        assert (facc["candidates"], facc["rescored"]) == (acc["candidates"], acc["rescored"]), tag
                if "ans" in calls:
                    got = t.analogy_answers(qf, names=names, bitlevel=bl, threshold=th)
                    assert np.array_equal(got, w2b.analogy_answers(vf, qf, bitlevel=bl, threshold=th)), tag
                for k in KS if "topk" in calls else ():
                    got = t.analogy_topk(qf, k, names=names, bitlevel=bl, threshold=th)
                    _same_lists(got, w2b.analogy_topk(vf, qf, k, bitlevel=bl, threshold=th), tag + " k %d" % k)
                    assert got[2]["packed"] == int(bit_route), (tag, got[2])
                    if bit_route:
                        want = w2b.analogy_topk(pf, qf, k, threshold=th)
                        _same_lists(got, want, tag + " k %d" % k)
                        assert _stats(got[2]) == _stats(want[2]), (tag, got[2], want[2])
                    if simt:
                        assert got[2]["simt"] == 1, (tag, got[2])
                for k in KS if "near" in calls else ():
                    got = t.nearest(wf, k, names=names, bitlevel=bl, threshold=th)
                    _same_lists(got, w2b.nearest(vf, wf, k, bitlevel=bl, threshold=th), tag + " nearest k %d" % k)
                    if bit_route:
                        want = w2b.nearest(pf, wf, k, threshold=th)
                        _same_lists(got, want, tag + " nearest k %d" % k)
                        assert _stats(got[2]) == _stats(want[2]), (tag, got[2], want[2])
    assert (t.table_checksum(), t.get_state()) == before


@pytest.mark.parametrize("bits", [0, 1, 2, 3, 5, 8])
@pytest.mark.parametrize("D", [4, 50, 800, 1023, 2048, 4096])
def test_crafted_tables_equal_the_file_round_trip(tmp_path, D, bits):
    u, v, names, qs = _crafted("mix", D, bits, seed=D * 10 + bits)
    t = _context(u, v, bits)
    try:
        vec = t.export()
        if bits != 3:  # (3 bits: every value quantises to a zero)
            assert not np.array_equal(vec.view(np.uint32), t.quantize(u, bits).view(np.uint32))
        qf, wf = str(tmp_path / "q.txt"), str(tmp_path / "w.txt")
        ac.write_questions(qf, qs)
        with open(wf, "w") as f:
            f.write("\n".join(names[:200] + ["missingword", names[5].lower()]) + "\n")
        _equal_to_round_trip(t, names, bits, qf, wf, str(tmp_path),
                             calls=("acc", "ans", "topk", "near") if D <= 800 else ("acc", "ans", "topk"))
    finally:
        t.close()


@pytest.mark.parametrize("kind,D,bits", [("all_equal", 32, 0), ("all_equal", 32, 1), ("all_equal", 32, 2),
                                         ("ties", 8, 1)])
def test_overflowing_tables_equal_the_file_round_trip(tmp_path, kind, D, bits):
    u, v, names, qs = _crafted(kind, D, bits, seed=7 + bits)
    t = _context(u, v, bits)
    try:
        qf, wf = str(tmp_path / "q.txt"), str(tmp_path / "w.txt")
        ac.write_questions(qf, qs)
        with open(wf, "w") as f:
            f.write("\n".join(names[:300]) + "\n")
        _equal_to_round_trip(t, names, bits, qf, wf, str(tmp_path), thresholds=())
        if kind == "all_equal":
            with _simt(False):
                _, acc = t.compute_accuracy(qf, names=names)
                st = t.analogy_topk(qf, 10, names=names)[2]
            assert acc["candidates"] > 1024 * acc["questions_seen"] and st["simt"] == 1
    finally:
        t.close()


# --------------------------------------------------------------------------------------- 3. a real trained context
def _corpus(d):
    path = zipf_corpus(os.path.join(d, "corpus.txt"), 60000, 3000, seed=5)
    c = w2b.Corpus(path, 5)
    words = c.words()
    rng = np.random.default_rng(1)
    qs = [[words[k] for k in rng.integers(1, min(len(words), 400), 4)] for _ in range(400)]
    qf, wf = os.path.join(d, "q.txt"), os.path.join(d, "w.txt")
    ac.write_questions(qf, qs)
    with open(wf, "w") as f:
        f.write("\n".join(words[1:150]) + "\n")
    return c, qf, wf


def _trained_equal(t, c, bits, qf, wf, d):
    """The four calls with names = the corpus's (names=None) against the round trip of export()."""
    vec = t.export()
    vf = os.path.join(d, "trained.bin")
    c.write_vectors(vf, vec, 1)
    pf = None
    if bits in (1, 2):
        pf = os.path.join(d, "trained.packed")
        c.write_packed(pf, vec, bits)
    for k in range(2):
        state = t.table_checksum(), t.get_state()
        text, _ = t.compute_accuracy(qf)
        assert text == w2b.compute_accuracy(vf, qf)[0]
        if pf:
            assert text == w2b.compute_accuracy_packed(pf, qf)[0]
        assert np.array_equal(t.analogy_answers(qf), w2b.analogy_answers(vf, qf))
        _same_lists(t.analogy_topk(qf, 10), w2b.analogy_topk(vf, qf, 10), "topk")
        _same_lists(t.nearest(wf, 10), w2b.nearest(vf, wf, 10), "nearest")
        assert (t.table_checksum(), t.get_state()) == state


@pytest.mark.parametrize("bits", [0, 1, 2])
def test_trained_context_equals_its_exported_file(tmp_path, bits):
    c, qf, wf = _corpus(str(tmp_path))
    kw = dict(size=48, window=5, negative=5, bitlevel=bits, threads=8, iter=2)
    t = w2b.Trainer(c, **kw)
    t.train_epoch()
    _trained_equal(t, c, bits, qf, wf, str(tmp_path))
    ck = str(tmp_path / "ckpt")
    t.checkpoint_save(ck, 1)
    t.close()
    t = w2b.Trainer(c, **kw)
    assert t.checkpoint_load(ck) == 1
    t.train_epoch()
    _trained_equal(t, c, bits, qf, wf, str(tmp_path))
    t.close()


def test_strict_training_after_an_evaluation_is_unchanged(tmp_path):
    c, qf, wf = _corpus(str(tmp_path))
    kw = dict(size=32, window=3, negative=4, bitlevel=1, threads=2, iter=2, mode=w2b.MODE_STRICT)
    runs = []
    for evaluate in (False, True):
        t = w2b.Trainer(c, **kw)
        t.train_epoch()
        if evaluate:
            t.compute_accuracy(qf)
            t.compute_accuracy(qf, bitlevel=2)
            t.analogy_answers(qf)
            t.analogy_topk(qf, 5)
            t.nearest(wf, 5, bitlevel=3)
        t.train_epoch()
        u, v = t.download_raw()
        runs.append((u.view(np.uint32).copy(), v.view(np.uint32).copy(), t.get_state()))
        t.close()
    (u0, v0, s0), (u1, v1, s1) = runs
    assert np.array_equal(u0, u1) and np.array_equal(v0, v1)
    assert np.float32(s0[0]).view(np.uint32) == np.float32(s1[0]).view(np.uint32) and s0[1] == s1[1]


# ----------------------------------------------------------------------------------------------------------- 4. CLI
def _tail2(text):
    return text.splitlines(keepends=True)[-2:]


def _cli_epochs(tmp_path, binary, threshold, gpus=1):
    c, qf, _ = _corpus(str(tmp_path))
    out = str(tmp_path / ("vec%d_%d" % (binary, gpus)))
    args = [TRAIN_CLI, "-train", str(tmp_path / "corpus.txt"), "-output", out, "-size", "32", "-iter", "2",
            "-bitlevel", "1", "-binary", str(binary), "-save-every-epoch", "1", "-eval", qf, "-threads", "8",
            "-gpus", str(gpus)]
    if threshold:
        args += ["-eval-threshold", str(threshold)]
    got = subprocess.run(args, capture_output=True, text=True, timeout=600)
    assert got.returncode == 0, got.stdout + got.stderr
    lines = got.stdout.split("\n")
    at = [i for i, l in enumerate(lines) if "Epoch Loss: " in l]
    assert len(at) == 2, got.stdout
    for epoch, i in enumerate(at):
        printed = [l + "\n" for l in lines[i + 1: i + 3]]
        want = subprocess.run([ACC_CLI, "%s_epoch%d" % (out, epoch), "0", str(threshold)], stdin=open(qf),
                              capture_output=True, text=True, timeout=300)
        assert want.returncode == 0
        assert printed == _tail2(want.stdout), (epoch, printed, want.stdout)
        assert printed[0].startswith("Total accuracy: ") and printed[1].startswith("Questions seen / total: ")


@pytest.mark.parametrize("binary,threshold", [(1, 0), (2, 300)])
def test_cli_prints_each_epochs_accuracy(tmp_path, binary, threshold):
    _cli_epochs(tmp_path, binary, threshold)


def test_cli_prints_each_epochs_accuracy_on_two_gpus(tmp_path):
    if w2b.device_count() < 2:
        pytest.skip("needs two GPUs")
    _cli_epochs(tmp_path, 1, 0, gpus=2)


# -------------------------------------------------------------------------------------------------------- 5. errors
def test_refused_calls_leave_the_context_usable(tmp_path):
    c, qf, wf = _corpus(str(tmp_path))
    names = c.words()
    t = w2b.Trainer(c, size=32, bitlevel=2, threads=4, iter=1, init=False)
    with pytest.raises(w2b.W2BError) as e:
        t.compute_accuracy(qf)
    assert e.value.code == ESTATE
    with pytest.raises(w2b.W2BError) as e:
        t.nearest(wf, 3)
    assert e.value.code == ESTATE
    t.init_tables()
    state = t.table_checksum(), t.get_state()
    n = C.c_int64()
    assert lib.w2b_ctx_compute_accuracy(t.h, None, 0, 0, qf.encode(), None, None, 0) == EINVAL
    assert t.table_checksum() == state[0]
    spaced = list(names)
    spaced[7] = "two words"
    for bad in (spaced, names[:7] + ["line\nbreak"] + names[8:]):
        with pytest.raises(w2b.W2BError) as e:
            t.analogy_answers(qf, names=bad)
        assert e.value.code == EINVAL
        assert (t.table_checksum(), t.get_state()) == state
    for k in (0, 1025):
        with pytest.raises(w2b.W2BError) as e:
            t.analogy_topk(qf, k)
        assert e.value.code == EINVAL
        assert (t.table_checksum(), t.get_state()) == state
    assert lib.w2b_ctx_analogy_answers(t.h, None, 0, 0, qf.encode(), None, 0, C.byref(n)) == EINVAL
    t.train_epoch()
    _trained_equal(t, c, 2, qf, wf, str(tmp_path))
    t.close()
