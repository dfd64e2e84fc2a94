"""oracle/philox.py, the host restatement of the device Philox streams (dropout keep bits, reparameterisation noise),
checked on the CPU: the Philox4x32-10 known-answer vectors of Salmon et al.'s Random123 distribution, the counter layout
of eb::Philox::gen, and the distribution of the two derived streams.  The device kernels are pinned to it in
tests/test_gpu_dense_model_kernels.py."""
import numpy as np

from oracle import philox as ph


def test_philox4x32_10_known_answers():
    # Random123 kat_vectors: philox4x32 10 rounds
    assert [int(x) for x in ph.philox4x32(0, 0, 0, 0, 0, 0)] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    got = ph.philox4x32(0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344, 0xA4093822, 0x299F31D0)
    assert [int(x) for x in got] == [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]
    got = ph.philox4x32(0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF)
    assert [int(x) for x in got] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


def test_gen_counter_layout_and_vectorisation():
    seed, ctr, att = 0x0123456789ABCDEF, (7 << 32) | 5, 9
    want = ph.philox4x32(5, 7, 9, ph.TAG, seed & 0xFFFFFFFF, seed >> 32)
    got = ph.gen(seed, [ctr], [att])
    assert [int(x[0]) for x in got] == [int(x) for x in want]
    many = ph.gen(seed, np.arange(100, dtype=np.uint64), np.full(100, 3, dtype=np.uint64))
    one = [ph.gen(seed, [c], [3]) for c in range(100)]
    for w in range(4):
        assert np.array_equal(many[w], np.array([int(o[w][0]) for o in one], dtype=np.uint32))


def test_keep_rate_and_independence():
    b, p = np.meshgrid(np.arange(400), np.arange(500), indexing="ij")
    for drop in (0.2, 0.5):
        k = ph.keep(1234, b, p, drop)
        n = k.size
        assert abs(k.mean() - (1 - drop)) < 5 * np.sqrt(drop * (1 - drop) / n)
        assert not np.array_equal(k[0], k[1]) and not np.array_equal(k, ph.keep(1235, b, p, drop))
    assert ph.keep(1234, b, p, 0.0).all()


def test_reparam_eps_is_standard_normal():
    e = ph.reparam_eps(42, 3, 200000)
    assert abs(e.mean()) < 5 / np.sqrt(e.size) and abs(e.var() - 1) < 5 * np.sqrt(2 / e.size)
    assert abs((e ** 4).mean() - 3) < 0.05                                    # normal kurtosis
    assert not np.array_equal(e[:1000], ph.reparam_eps(42, 4, 1000))


def test_csr_keep_mask_places_the_bits_of_each_row():
    indptr = np.array([0, 3, 3, 5], np.int64); indices = np.array([1, 4, 6, 0, 6], np.int32)
    K = ph.csr_keep_mask(9, indptr, indices, [2, 0, 1], 8, 0.5)
    assert K.shape == (3, 8) and not K[2].any()
    assert np.array_equal(K[0, [0, 6]], ph.keep(9, 0, np.arange(2), 0.5).astype(float))
    assert np.array_equal(K[1, [1, 4, 6]], ph.keep(9, 1, np.arange(3), 0.5).astype(float))
    assert not K[0, [1, 2, 3, 4, 5, 7]].any()
