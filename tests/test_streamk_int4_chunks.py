"""CPU model-check of the INT4 stream-K code chunks (csrc/gemm_streamk.cuh, SkW4Cfg and the W4 producer / converter branches).

One thread requests chunks of up to four k-blocks of one tile into a ring of SK_W4_SLOTS slots; the converter warps walk the
units and must agree on where every chunk starts; a slot is requested again only after the converters have finished its previous
chunk.  Checked over the partitions of tests/test_streamk_protocol.py: the two sides cut the same chunks, every chunk lies in one
tile and within 16 KB, every unit of the range is covered once in order, and the producer's order of waits never deadlocks (the
chunk of unit `it` is requested before the producer blocks on the stage of `it`, and its slot's previous chunk only holds
earlier units).
"""
import random

import pytest

from tests.test_streamk_protocol import SHAPES, SK_BN, TG_BK, first

CHUNK_KB, SLOTS, STAGES = 4, 4, 5


def producer_chunks(u_begin, n_it, num_k):
    """issue_chunk: (first iteration, length) of every chunk of a range."""
    out, it = [], 0
    while it < n_it:
        kb = (u_begin + it) % num_k
        n = min(CHUNK_KB, num_k - kb, n_it - it)
        out.append((it, n))
        it += n
    return out


def converter_starts(u_begin, n_it, num_k):
    """The converter's boundary rule: kb == 0, four k-blocks done, or the first unit."""
    starts, pos = [], CHUNK_KB
    for it in range(n_it):
        kb = (u_begin + it) % num_k
        if kb == 0 or pos == CHUNK_KB or it == 0:
            starts.append(it)
            pos = 0
        pos += 1
    return starts


@pytest.mark.parametrize("G", [132, 148, 7])
def test_both_sides_cut_the_same_chunks(G):
    for N, K in SHAPES:
        if K % 128:
            continue
        num_n, num_k = N // SK_BN, K // TG_BK
        total = num_n * num_k
        grid = min(G, total)
        for c in range(grid):
            u0, u1 = first(total, grid, c), first(total, grid, c + 1)
            chunks = producer_chunks(u0, u1 - u0, num_k)
            assert [it for it, _ in chunks] == converter_starts(u0, u1 - u0, num_k), (N, K, c)
            assert sum(n for _, n in chunks) == u1 - u0
            for it, n in chunks:
                assert 1 <= n <= CHUNK_KB and (u0 + it) // num_k == (u0 + it + n - 1) // num_k, "a chunk must lie in one tile"
                assert SK_BN * n * TG_BK // 2 <= 16384


@pytest.mark.parametrize("seed", range(8))
def test_ring_order_never_deadlocks(seed):
    """Producer, converters and consumers of one CTA advance in random order, each blocking exactly where the kernel blocks."""
    r = random.Random(seed)
    num_k = r.choice([2, 3, 4, 6, 12, 64, 448])
    n_it = r.randint(1, 200)
    u0 = r.randint(0, num_k * 5)
    chunks = producer_chunks(u0, n_it, num_k)
    chunk_of = {}
    for ci, (it, n) in enumerate(chunks):
        for j in range(it, it + n):
            chunk_of[j] = ci
    issued, a_done, conv_done, cons_done = 0, 0, 0, 0  # chunks requested; units whose A / W' / MMA are done

    def converted_chunks():
        return sum(1 for ci, (it, n) in enumerate(chunks) if it + n <= conv_done)

    steps = 0
    while cons_done < n_it:
        steps += 1
        assert steps < 100000, "deadlock"
        who = r.choice(["prod", "conv", "cons"])
        if who == "prod" and a_done < n_it:
            it = a_done
            if issued <= chunk_of[it]:  # must request the chunk of `it` (blocking on its slot)
                if issued < converted_chunks() + SLOTS:
                    issued += 1
                continue
            while issued < len(chunks) and issued < converted_chunks() + SLOTS and r.random() < 0.5:  # opportunistic
                issued += 1
            if it - STAGES < cons_done:  # stage of `it` free
                a_done += 1
        elif who == "conv" and conv_done < n_it:
            it = conv_done
            if chunk_of[it] < issued and it - STAGES < cons_done:  # chunk landed and stage free
                conv_done += 1
        elif who == "cons" and cons_done < n_it:
            if cons_done < a_done and cons_done < conv_done:
                cons_done += 1
    assert issued == len(chunks)
