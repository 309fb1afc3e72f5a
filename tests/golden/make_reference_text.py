"""Generates tests/golden/reference_text_b0.txt and reference_text_b1.txt: text vector files (-binary 0) written by
the UNMODIFIED reference (oracle/_ref/word2bits, built by oracle/Makefile) from the golden corpus, one with fp32 values
(-bitlevel 0, D = 12) and one on the 1-bit levels (-bitlevel 1, D = 8).  One training thread, so the files do not
depend on scheduling.  The text reader's tests read them as the files users get from the reference.

    python tests/golden/make_reference_text.py"""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REFBIN = os.path.join(ROOT, "oracle", "_ref", "word2bits")
FILES = {"reference_text_b0.txt": ("0", "12"), "reference_text_b1.txt": ("1", "8")}


def main():
    assert os.path.exists(REFBIN), "build oracle/_ref first"
    for name, (bits, size) in FILES.items():
        out = os.path.join(HERE, name)
        subprocess.run([REFBIN, "-train", os.path.join(HERE, "golden_corpus.txt"), "-output", out, "-size", size,
                        "-bitlevel", bits, "-binary", "0", "-threads", "1", "-iter", "2", "-min-count", "3",
                        "-window", "3", "-negative", "4"], check=True, capture_output=True)
        print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
