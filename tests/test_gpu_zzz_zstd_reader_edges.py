"""GPU: the backward bit reader's edge corpus of tests/test_zstd_reader_edges.py (streams at every offset mod 8, in the source's first
words and ending on its last byte, sizes around the window and the words in flight, literal and sequence counts one off) through
Codec.decompress, frame by frame and as one stream, against the oracle decoder's bytes or verdict."""
import pytest

from test_zstd_crafted import CHECKSUM, CORRUPT, UNSUPPORTED, oracle_verdict
from test_zstd_reader_edges import reader_corpus

pytestmark = pytest.mark.gpu

ERR = {CORRUPT: -5, UNSUPPORTED: -6, CHECKSUM: -8}


@pytest.fixture(scope="module")
def corpus():
    return [(name, s, oracle_verdict(s, 1 << 18)) for name, s in reader_corpus()]


@pytest.mark.parametrize("dec_jump", [0, 2])
def test_reader_edges_match_the_oracle(pkg, corpus, dec_jump):
    c = pkg.Codec(0, dec_jump=dec_jump)
    try:
        for name, stream, want in corpus:
            if isinstance(want, bytes):
                assert c.decompress(stream, max_size=1 << 18) == want, (name, dec_jump)
            else:
                with pytest.raises(Exception) as e:
                    c.decompress(stream, max_size=1 << 18)
                assert getattr(e.value, "code", None) == ERR[want], (name, dec_jump, e.value)
    finally:
        c.close()


def test_valid_reader_edges_as_one_stream(pkg, corpus):
    """every valid frame in one call: thousands of streams in the same launches, their words in flight side by side"""
    valid = [(s, want) for _, s, want in corpus if isinstance(want, bytes)]
    stream = b"".join(s for s, _ in valid); plain = b"".join(w for _, w in valid)
    c = pkg.Codec(0)
    try:
        assert c.decompress(stream, max_size=len(plain)) == plain
    finally:
        c.close()
