"""Host model of the tagged hand-off of k_gn_persistent (ct_icp_b200/csrc/icp_gn.cu, tagged_words.cuh).

Every 8-byte word carries 32 payload bits and a 32-bit tag. A gather CTA stores its partial row of iteration `it` as 2 x kAcc
words tagged `base + it` (each double as its low and high half); the solver CTA's warps consume the rows in a fixed order,
each as soon as all its words carry that tag, and publish the next pose as tagged words; warp 0 of a gather CTA polls those
until every word carries `base + it + 1`. The host (IcpSolver::ReserveLoopTags) hands out `num_iters + 1` tags per launch and
zeroes the words when the counter would wrap.

Modelled with real threads and random delays, the writers storing a row or the pose word by word in a random order, so a
reader can see a torn mix of old and new words. Checked: the solver never adds a word of another iteration or launch, the
streamed sum equals gn_reduce_rows's order bit for bit, the one-buffer invariant holds, and early convergence, the last
iteration and a row time-out terminate every thread."""
import math
import random
import struct
import threading
import time

import pytest

K_ACC = 96            # kAcc
K_ROW_WORDS = 2 * K_ACC
K_GATHER_WARPS = 16   # CTICP_GATHER_WARPS
K_POSE_WORDS = 36     # 2 x kPosePairs
MASK32 = 0xffffffff


def split_double(d):
    """the two 32-bit halves of a double, low half first (tagged_store_double)"""
    lo, hi = struct.unpack("<II", struct.pack("<d", d))
    return lo, hi


def join_double(lo, hi):
    """pair_double"""
    return struct.unpack("<d", struct.pack("<II", lo, hi))[0]


def word(tag, payload):
    return (tag << 32) | payload


def word_tag(w):
    return w >> 32


class Tags:
    """IcpSolver::ReserveLoopTags: a launch reserves num_iters + 1 tags; tag 0 is never handed out; before the counter would
    wrap, the words are zeroed and it restarts at 1."""

    def __init__(self, start=1):
        self.next = start

    def reserve(self, num_iters, buffers):
        span = max(num_iters, 0) + 1
        if self.next + span > MASK32:
            for buf in buffers:
                for i in range(len(buf)):
                    buf[i] = 0
            self.next = 1
        base = self.next
        self.next += span
        assert self.next <= MASK32
        return base


def row_values(launch, c, it):
    """the partial row gather CTA c writes in iteration it of a launch: includes values whose halves look alike"""
    rng = random.Random(launch * 1000003 + c * 1009 + it)
    vals = [rng.uniform(-1e3, 1e3) * 10 ** rng.randint(-30, 30) for _ in range(K_ACC)]
    vals[0] = -0.0
    vals[1] = 5e-324 * (c + 1)   # subnormal
    vals[2] = float(it)
    return vals


def pose_values(launch, it):
    """stand-in for the pose of iteration it: 16 doubles and two ints (GnPose), then `done`"""
    return [launch + it / 8.0 + k for k in range(16)]


class _Launch:
    def __init__(self, rows, pose, base, launch, gather_ctas, num_iters, done_after, dead_cta, seed, timeout):
        self.rows, self.pose, self.base, self.launch = rows, pose, base, launch
        self.G, self.I, self.done_after, self.dead_cta = gather_ctas, num_iters, done_after, dead_cta
        self.rng = random.Random(seed)
        self.lock = threading.Lock()
        self.timeout = timeout
        self.errors = []
        self.sums = []
        self.consumed = [-1] * gather_ctas    # last iteration whose row the solver consumed, per gather CTA
        self.pose_read = [0] * gather_ctas    # iteration whose pose each gather CTA read last
        self.failed = 0

    def jitter(self, p=0.05, scale=2e-4):
        with self.lock:
            r = self.rng.random()
            d = self.rng.random() * scale
        if r < p:
            time.sleep(d)

    def store_words(self, buf, offset, words):
        """one thread's (or CTA's) stores of a block of words, in a random order with delays in between"""
        with self.lock:
            order = list(range(len(words)))
            self.rng.shuffle(order)
        for i in order:
            buf[offset + i] = words[i]
            self.jitter(0.02, 5e-5)

    # ---- gather CTA ---------------------------------------------------------------------------------------------------
    def gather(self, c):
        for it in range(self.I):
            tag = self.base + it
            if it > 0:
                deadline = time.time() + self.timeout
                while True:   # gn_fetch_pose: every pose word carries the tag
                    snap = list(self.pose[:K_POSE_WORDS])
                    if all(word_tag(w) == tag for w in snap):
                        break
                    if time.time() > deadline:
                        self.errors.append("gather %d: pose of %d never arrived" % (c, it))
                        return
                    time.sleep(0)
                vals = [join_double(snap[2 * k] & MASK32, snap[2 * k + 1] & MASK32) for k in range(16)]
                done = snap[34] & MASK32
                if done:
                    return
                if vals != pose_values(self.launch, it):
                    self.errors.append("gather %d read a pose of another iteration in %d" % (c, it))
                self.pose_read[c] = it
                if self.consumed[c] != it - 1:   # the one-buffer invariant, gather side
                    self.errors.append("gather %d rewrites its row of %d before the solver consumed it" % (c, it - 1))
            if c == self.dead_cta and it == 1:
                return   # a CTA that never delivers its row
            self.jitter(0.3, 1e-3)
            words = []
            for v in row_values(self.launch, c, it):
                lo, hi = split_double(v)
                words += [word(tag, lo), word(tag, hi)]
            self.store_words(self.rows, c * K_ROW_WORDS, words)
            if it == self.I - 1:
                return

    # ---- solver CTA ---------------------------------------------------------------------------------------------------
    def reduce(self, it):
        """gn_reduce_tagged_rows: per warp, rows w, w + 16, … in order, a row added once all its words carry the tag; then
        the per-warp sums in warp order. Returns None on time-out."""
        tag = self.base + it
        deadline = time.time() + self.timeout
        warp_sums = []
        for w in range(K_GATHER_WARPS):
            acc = [0.0] * K_ACC
            for b in range(w, self.G, K_GATHER_WARPS):
                while True:
                    snap = list(self.rows[b * K_ROW_WORDS:(b + 1) * K_ROW_WORDS])
                    if all(word_tag(x) == tag for x in snap):
                        break
                    if time.time() > deadline:
                        return None
                    time.sleep(0)
                vals = [join_double(snap[2 * k] & MASK32, snap[2 * k + 1] & MASK32) for k in range(K_ACC)]
                want = row_values(self.launch, b, it)
                if [split_double(v) for v in vals] != [split_double(v) for v in want]:
                    self.errors.append("solver added a word of another iteration or launch (row %d, it %d)" % (b, it))
                for k in range(K_ACC):
                    acc[k] += vals[k]
                self.consumed[b] = it
            warp_sums.append(acc)
        total = []
        for k in range(K_ACC):
            s = 0.0
            for w in range(K_GATHER_WARPS):
                s += warp_sums[w][k]
            total.append(s)
        return total

    def publish(self, it, done):
        """gn_publish_pose: the pose words of iteration it, tagged base + it"""
        tag = self.base + it
        words = []
        for v in pose_values(self.launch, it):
            lo, hi = split_double(v)
            words += [word(tag, lo), word(tag, hi)]
        words += [word(tag, 0), word(tag, 1), word(tag, 1 if done else 0), word(tag, 0)]
        assert len(words) == K_POSE_WORDS
        self.store_words(self.pose, 0, words)

    def solver(self):
        done = False
        for it in range(self.I):
            if done:
                break
            total = self.reduce(it)
            if total is None:   # a row never arrived: failed = 2, done = 1 in the pose words of the next iteration
                self.failed = 2
                self.publish(it + 1, True)
                return
            self.sums.append(total)
            self.jitter(0.3, 1e-3)
            done = self.done_after is not None and it + 1 >= self.done_after
            if it + 1 < self.I:
                for c in range(self.G):   # the one-buffer invariant, solver side
                    if self.pose_read[c] < it:
                        self.errors.append("solver rewrites the pose of %d before gather %d read it" % (it, c))
                self.publish(it + 1, done)


def reference_sums(launch, gather_ctas, iters):
    """gn_reduce_rows's order on the values themselves"""
    out = []
    for it in range(iters):
        warp_sums = []
        for w in range(K_GATHER_WARPS):
            acc = [0.0] * K_ACC
            for b in range(w, gather_ctas, K_GATHER_WARPS):
                vals = row_values(launch, b, it)
                for k in range(K_ACC):
                    acc[k] += vals[k]
            warp_sums.append(acc)
        total = []
        for k in range(K_ACC):
            s = 0.0
            for w in range(K_GATHER_WARPS):
                s += warp_sums[w][k]
            total.append(s)
        out.append(total)
    return out


def run_launch(rows, pose, tags, launch, gather_ctas, num_iters, done_after=None, dead_cta=None, seed=0, timeout=10.0):
    base = tags.reserve(num_iters, [rows, pose])
    L = _Launch(rows, pose, base, launch, gather_ctas, num_iters, done_after, dead_cta, seed, timeout)
    threads = [threading.Thread(target=L.gather, args=(c,)) for c in range(gather_ctas)] + [threading.Thread(target=L.solver)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(60)
    assert not any(t.is_alive() for t in threads), "a thread never terminated"
    return L


def same_bits(a, b):
    return [split_double(x) for x in a] == [split_double(x) for x in b]


@pytest.mark.parametrize("gather_ctas,iters,done_after,seed", [(7, 4, None, 1), (20, 3, None, 2), (37, 3, 1, 3),
                                                               (3, 5, 2, 4), (100, 2, None, 5)])
def test_two_launches_share_the_buffers(gather_ctas, iters, done_after, seed):
    rows = [0] * (K_ROW_WORDS * gather_ctas)
    pose = [0] * 48
    tags = Tags()
    # a second launch with another iteration count reuses every word of the first
    for launch, n_it in ((1, iters), (2, iters + 2)):
        L = run_launch(rows, pose, tags, launch, gather_ctas, n_it, done_after, seed=seed * 10 + launch)
        assert not L.errors, L.errors[:3]
        ran = n_it if done_after is None else min(n_it, done_after)
        assert len(L.sums) == ran
        ref = reference_sums(launch, gather_ctas, ran)
        for it in range(ran):
            assert same_bits(L.sums[it], ref[it]), "streamed sum differs from gn_reduce_rows's order at %d" % it


def test_wrap_of_the_tag_counter_zeroes_the_words():
    rows = [0] * (K_ROW_WORDS * 9)
    pose = [0] * 48
    tags = Tags(start=MASK32 - 6)
    L = run_launch(rows, pose, tags, 1, 9, 4, seed=7)   # tags 2^32 - 7 .. 2^32 - 3
    assert not L.errors and len(L.sums) == 4
    assert tags.next == MASK32 - 1
    L = run_launch(rows, pose, tags, 2, 9, 3, seed=8)   # does not fit: words zeroed, tags restart at 1
    assert L.base == 1 and tags.next == 5
    assert not L.errors and len(L.sums) == 3
    ref = reference_sums(2, 9, 3)
    assert all(same_bits(L.sums[i], ref[i]) for i in range(3))


def test_row_time_out_releases_every_gather_cta():
    rows = [0] * (K_ROW_WORDS * 6)
    pose = [0] * 48
    L = run_launch(rows, pose, Tags(), 1, 6, 5, dead_cta=3, seed=11, timeout=0.5)
    assert L.failed == 2
    assert len(L.sums) == 1   # iteration 0 completed, iteration 1 timed out
    assert not [e for e in L.errors if "another" in e], L.errors


def test_stale_rows_of_the_previous_launch_are_never_added():
    """A row left by launch 1 at a higher iteration than launch 2 has reached carries a tag launch 2 never waits for."""
    rows = [0] * (K_ROW_WORDS * 4)
    pose = [0] * 48
    tags = Tags()
    b1 = tags.reserve(6, [rows, pose])
    b2 = tags.reserve(3, [rows, pose])
    used1 = {b1 + it for it in range(6)}
    used2 = {b2 + it for it in range(3)}
    assert not used1 & used2 and 0 not in used1 | used2


@pytest.mark.parametrize("d", [0.0, -0.0, 5e-324, -5e-324, 2.2250738585072009e-308, 1.0, -1.5e300, math.inf, -math.inf,
                               math.pi, 1e-310])
def test_double_halves_round_trip_exactly(d):
    for tag in (1, 0x7fffffff, MASK32):
        lo, hi = split_double(d)
        w_lo, w_hi = word(tag, lo), word(tag, hi)
        assert word_tag(w_lo) == tag and word_tag(w_hi) == tag
        back = join_double(w_lo & MASK32, w_hi & MASK32)
        assert struct.pack("<d", back) == struct.pack("<d", d)


def test_nan_payloads_round_trip_exactly():
    for bits in (0x7ff8000000000000, 0xfff8000000000001, 0x7ff0000000000001, 0x7fffffffffffffff):
        d = struct.unpack("<d", struct.pack("<Q", bits))[0]
        lo, hi = split_double(d)
        back = join_double(word(9, lo) & MASK32, word(9, hi) & MASK32)
        assert struct.unpack("<Q", struct.pack("<d", back))[0] == bits
