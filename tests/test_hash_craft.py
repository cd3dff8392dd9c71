"""CPU: the collision toolkit of tests/hash_craft.py — the inverses round-trip, every constructor's output really
collides under the restated hash, and the constructors are deterministic for a seed."""
import numpy as np

import hash_craft as H


def test_hash64_inverse_round_trips():
    rng = np.random.default_rng(0)
    xs = [0, 1, H.M64, 1 << 63] + [int(v) for v in rng.integers(0, 1 << 63, 200, dtype=np.uint64)]
    for x in xs:
        assert H.hash64_inv(H.hash64(x)) == x and H.hash64(H.hash64_inv(x)) == x
    a = np.asarray(xs, dtype=np.uint64)
    assert [int(v) for v in H.hash64_np(a)] == [H.hash64(x) for x in xs]
    # the murmur3 finaliser's known value
    assert H.hash64(1) == 0xb456bcfc34c2cb2c


def test_hash_bytes_step_inverse_and_tail():
    rng = np.random.default_rng(1)
    for _ in range(100):
        h, w = (int(v) for v in rng.integers(0, 1 << 63, 2, dtype=np.uint64))
        assert H.hb_step_inv(H.hb_step(h, w)) == h ^ w
    # a tail is one zero-padded step; the length is in the seed, so padding does not collide
    assert H.hash_bytes(b"abc") != H.hash_bytes(b"abc\0")
    assert H.hash_bytes(b"abcdefgh" * 2) == H.hb_step(H.hb_step(H.HB_SEED ^ 16, int.from_bytes(b"abcdefgh", "little")),
                                                      int.from_bytes(b"abcdefgh", "little"))


def _merges(n=600, seed=1):
    rng = np.random.default_rng(seed)
    return np.stack([rng.integers(0, 256 + i, 2) for i in range(n)]).astype(np.int32)


def test_merges_collision():
    m = _merges()
    for r in (0, 3, 100, 598):
        m2 = H.merges_collision(m, r, seed=r)
        assert m2.shape == m.shape and not np.array_equal(m2, m)
        assert np.array_equal(np.nonzero((m2 != m).any(1))[0][:1], [r])
        assert ((m2 != m).any(1)).sum() <= 2 and (m2 >= 0).all()
        assert H.hash_bytes(m2.astype("<i4").tobytes()) == H.hash_bytes(m.astype("<i4").tobytes())
        assert np.array_equal(H.merges_collision(m, r, seed=r), m2)


def test_perm_collision():
    perm = np.random.default_rng(2).permutation(256).astype(np.uint8)
    for r in (0, 17, 30):
        p2 = H.perm_collision(perm, r, seed=r)
        assert p2.dtype == np.uint8 and p2.size == 256 and not np.array_equal(p2, perm)
        assert H.hash_bytes(p2.tobytes()) == H.hash_bytes(perm.tobytes())
        assert np.array_equal(H.perm_collision(perm, r, seed=r), p2)


def test_specials_collision():
    A = [(b"<|a|>", 100257), (b"<|b|>", 100258)]
    B = H.specials_collision_search(A, lambda t: [b"<|c%02d|>" % t, b"<|d|>"])
    assert B == [(b"<|c00|>", 395947165), (b"<|d|>", 1135673233)]
    assert H.spec_hash(B) == H.spec_hash(A) and B != A
    C = H.specials_collision_search([(b"hello", 100300), (b"<|e|>", 100301)], lambda t: [b"<|f%03d|>" % t, b"<|g|>"])
    assert H.spec_hash(C) == H.spec_hash([(b"hello", 100300), (b"<|e|>", 100301)])


def test_e2_tag_collision_and_cluster():
    a = b"abcdefgh" * 2
    b = H.e2_collision(a, b"zzzzzzzz")
    assert b != a and len(b) == 16 and b[:8] == b"zzzzzzzz" and H.e2_tag(a) == H.e2_tag(b)
    for n in (8, 24, 48):
        prefix = bytes(range(65, 65 + n - 8))
        t = (0x123456789 << 20) | 5
        assert H.e2_tag(H.e2_chunk_for_tag(prefix, t)) == t | 1
    cl = H.e2_cluster(30, 12, 4095, prefix=b" cluster", seed=3)
    assert len(set(cl)) == 30 and all(H.e2_home(H.e2_tag(c), 12) == 4095 for c in cl)
    assert len({H.e2_tag(c) for c in cl}) == 30
    assert H.e2_cluster(30, 12, 4095, prefix=b" cluster", seed=3) == cl


def test_dd_collision():
    a, b = H.dd_collision(3, seed=0)
    assert a != b and len(a) == len(b) == 12
    assert H.dd_key(a) == H.dd_key(b)
    assert H.dd_tag(H.dd_key(a)) == H.dd_tag(H.dd_key(b)) and H.dd_home(H.dd_key(a), 20) == H.dd_home(H.dd_key(b), 20)
    assert H.dd_collision(3, seed=0) == (a, b)
    # the additive steps: a 4-byte tail is zero padded
    assert H.dd_key(b"ab") != H.dd_key(b"ab\0\0")


def test_dd_cluster():
    def make(rng, n):
        return [b" " + bytes(rng.integers(97, 123, 6).astype(np.uint8)) for _ in range(n)]
    cl = H.dd_cluster(70, 12, 7, make, seed=4, batch=4096)
    assert len(set(cl)) == 70 and all(H.dd_home(H.dd_key(c), 12) == 7 for c in cl)
    assert H.dd_cluster(70, 12, 7, make, seed=4, batch=4096) == cl


def test_pair_homes():
    mask = 1023
    cl = H.pair_cluster(40, mask, mask, seed=5)
    assert len(set(cl)) == 40 and all(H.table_home(a, b, mask) == mask for a, b in cl)
    assert all(a < (1 << 16) and b < (1 << 16) for a, b in cl)
    assert H.pair_cluster(40, mask, mask, seed=5) == cl
    dense = H.byte_pairs_in_slot(100, H.hist_dense_home)
    assert len(dense) >= 10 and all(((((a << 8) | b) * 2654435761) % (1 << 32)) >> 20 == 100 for a, b in dense)
    hh = H.byte_pairs_in_slot(9, H.hist_hash_home)
    assert len(hh) >= 8 and all(H.hash64((a << 32) | b) % 2048 == 9 for a, b in hh)
