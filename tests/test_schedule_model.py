"""
CPU tier: the balanced persistent schedule of the fused kernels (TileSched, sched_* in
setk_b200/csrc/stft_tile.cuh; fused_schedule in stft_cov_fused.cu, which sets it up for the
fused STFT + covariance and the fused apply + iSTFT alike), restated in Python and
checked over random batch shapes: every (utterance, tile) pair is owned by exactly one CTA,
a CTA's partial-sum slot index stays below the reserved slot count, and cov_finalize_kernel's
"slots used by utterance b" formula names exactly the slots that were written.
(The kernels themselves run this schedule in tests/test_emu_kernels.py and on the GPU.)
"""
import random


def tiles_of(frames, TT):
    return (frames + TT - 1) // TT if frames > 0 else 1          # sched_tiles_of


def slots_of(n_ctas, B):                                         # sched_slots
    s = (n_ctas + B - 1) // B + 3
    return 4 if s < 4 else (18 if s > 18 else s)


def min_quota(tiles_max, slots):                                 # sched_min_quota
    return (tiles_max + slots - 3) // (slots - 2)


def grid(total_max, n_ctas, mq):                                 # sched_grid
    q = max((total_max + n_ctas - 1) // n_ctas, mq, 1)
    return (total_max + q - 1) // q


def test_every_tile_owned_once_and_slots_bounded():
    rnd = random.Random(1)
    for _ in range(4000):
        TT = rnd.choice([4, 5])
        G = rnd.choice([2, 16, 132, 148, 264, 296])
        B = rnd.choice([1, 2, 3, 7, 37, 64, 256, 300, 1000])
        Tmax = rnd.choice([1, 2, 5, 63, 626, 6251])
        tiles_max = tiles_of(Tmax, TT)
        S = slots_of(G, B)
        mq = min_quota(tiles_max, S)
        n_ctas = grid(B * tiles_max, G, mq)
        mode = rnd.choice(["uniform", "ragged", "tiny"])
        if mode == "uniform":
            frames = [Tmax] * B
        elif mode == "ragged":
            frames = [rnd.randint(0, Tmax) for _ in range(B)]
        else:
            frames = [rnd.choice([0, 1, Tmax]) for _ in range(B)]
        prefix = [0]
        for f in frames:
            prefix.append(prefix[-1] + tiles_of(f, TT))
        total = prefix[-1]
        q = max((total + n_ctas - 1) // n_ctas, mq, 1)           # sched_quota (device side)
        assert n_ctas * q >= total
        owners = [0] * total
        written = {}
        for g in range(n_ctas):
            cur, hi = g * q, min(g * q + q, total)
            if cur >= hi:
                continue
            b = max(i for i in range(B) if prefix[i] <= cur)     # sched_find
            while cur < hi:
                while prefix[b + 1] <= cur:
                    b += 1
                seg_end = min(hi, prefix[b + 1])
                slot = g - prefix[b] // q
                assert 0 <= slot < S, (slot, S, B, G, Tmax, mode)
                written.setdefault(b, set()).add(slot)
                for x in range(cur, seg_end):
                    owners[x] += 1
                cur = seg_end
        assert all(c == 1 for c in owners)
        for b in range(B):
            n_used = (prefix[b + 1] - 1) // q - prefix[b] // q + 1   # cov_finalize_kernel
            assert written.get(b, set()) == set(range(n_used)), (b, written.get(b), n_used)
