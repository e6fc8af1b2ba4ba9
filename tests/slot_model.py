"""numpy model of K1t2's slot layout (csrc/apo_kernels.h, apo_tuple.cu k_slot_plane / k_tuple_slots, apo_abi.cu
build_twin_t2) and of the shared-memory wavefronts its gather needs.

The copy's dictionary is in frequency order.  The h most frequent entries get 16 slots each (entry e, copy k: slot 16 e + k,
bank pair k), slot 16 h holds zero, entries [h, end) one slot each (e + 15 h + 1), entries >= end none: their evaluations
read the zero slot and are listed.  Per half-warp instruction of K1t2 (evaluations b * 128 + 8 l + q, l < 16) the
single-slot lanes claim their bank pairs first, then each distinct hot entry takes its own lane's bank pair if free, else the
lowest free one."""
import numpy as np

REP = 16
SLOT_H = 512
HOT_MAX = 28672          # K1t2's shared-memory head, in slots
SHARE = 64               # a list may hold at most 1/64 of the evaluations


def slot_end(n, h):
    return min(n, 65535 - (REP - 1) * h)


def choose_h(counts, N):
    """build_twin_t2's choice of h from the dictionary's counts (frequency order)"""
    n = len(counts)
    c16 = np.asarray(counts[:65536], np.uint64)
    h = min(SLOT_H, n)
    while True:
        end = slot_end(n, h)
        ny = int(c16[end:].sum())
        if ny * SHARE <= N or h == 0:
            return h, end
        h //= 2


def slot_table(tval, h, end):
    """the slot-order table of the entry-order one"""
    tval = np.asarray(tval, np.int64)
    z = REP * h
    i = np.arange(end + (REP - 1) * h + 1)
    out = np.zeros(len(i), np.int64)
    out[:z] = tval[i[:z] // REP]
    out[z + 1:] = tval[i[z + 1:] - (REP - 1) * h - 1]
    return out


def slot_plane(idx, h, end):
    """slots of the full indices idx [C][T] (uint32)"""
    idx = np.asarray(idx, np.int64)
    C, T = idx.shape
    nb = (T + 127) // 128
    full = np.full((C, nb * 128), -1, np.int64)
    full[:, :T] = idx
    g = full.reshape(C, nb, 16, 8).transpose(0, 1, 3, 2).reshape(-1, 16)      # [group][lane l]: b * 128 + 8 l + q
    valid = g >= 0
    hot = valid & (g < h)
    cold_slot = np.where(g < end, g + (REP - 1) * h + 1, REP * h)
    used = np.zeros(len(g), np.int64)
    for l in range(16):
        m = valid[:, l] & ~hot[:, l]
        used[m] |= 1 << (cold_slot[m, l] & 15)
    bp = np.full(g.shape, -1, np.int64)
    for l in range(16):
        todo = hot[:, l].copy()
        for m in range(l):
            same = todo & hot[:, m] & (g[:, m] == g[:, l])
            bp[same, l] = bp[same, m]
            todo &= ~same
        free = ~used & 0xFFFF
        own = (free >> l) & 1 == 1
        low = np.zeros(len(g), np.int64)
        for k in range(15, -1, -1):                  # lowest free bank pair
            low = np.where((free >> k) & 1 == 1, k, low)
        pick = np.where(own | (free == 0), l, low)
        bp[todo, l] = pick[todo]
        used[todo] |= 1 << pick[todo]
    slots = np.where(hot, REP * g + bp, cold_slot)
    out = slots.reshape(C, nb, 8, 16).transpose(0, 1, 3, 2).reshape(C, nb * 128)[:, :T]
    return out.astype(np.uint16)


def lists(idx, end):
    """(exceptions, evaluations of entries [end, 2^16)) as [(row, position, full index)]"""
    idx = np.asarray(idx, np.int64)
    ex = np.argwhere(idx >= 65536)
    lo = np.argwhere((idx >= end) & (idx < 65536))
    return [(int(c), int(t), int(idx[c, t])) for c, t in ex], [(int(c), int(t), int(idx[c, t])) for c, t in lo]


def row_sums(idx, slots, tval, h, end):
    """what K1t2 sums per row: the slot plane through the slot-order table, plus both lists from the entry-order table"""
    sval = slot_table(tval, h, end)
    s = sval[slots.astype(np.int64)].sum(axis=1, dtype=np.int64)
    for lst in lists(idx, end):
        for c, _, full in lst:
            s[c] += tval[full]
    return s


def wavefronts(slots, hot=HOT_MAX, first=0):
    """the wavefront model of K1t2's LDS.64 over whole 256-evaluation warp steps from `first`: per warp instruction (lanes
    8 apart) the largest number of distinct 4-byte words any bank serves, counted over the warp and summed over its two
    half-warps; and the mean number of lanes per warp instruction whose slot is past the shared-memory head"""
    s = np.asarray(slots, np.int64)[:, first:]
    C, T = s.shape
    nw = T // 256
    s = s[:, :nw * 256].reshape(C * nw, 32, 8).transpose(0, 2, 1).reshape(-1, 32)   # [instruction][lane]
    tail = s >= hot
    words = np.stack([2 * s, 2 * s + 1], axis=-1)                                       # [instr][lane][2] word addresses
    words[tail] = -1                                                                    # predicated off: the L2 path

    def worst(w):
        w = w.reshape(len(w), -1)
        banks = w & 31
        best = np.zeros(len(w), np.int64)
        for b in range(32):
            wb = np.where(banks == b, w, -1)
            wb.sort(axis=1)
            distinct = ((wb[:, 1:] != wb[:, :-1]) & (wb[:, 1:] >= 0)).sum(axis=1) + (wb[:, 0] >= 0)
            best = np.maximum(best, distinct)
        return best

    warp = worst(words)
    half = worst(words[:, :16]) + worst(words[:, 16:])
    return {"warp": float(warp.mean()), "half_warps": float(half.mean()), "tail_lanes": float(tail.sum(axis=1).mean())}
