"""CPU: the synchronisation protocol of the GEMM's alternating schedule, simulated over mbarrier semantics.

The ring arithmetic is the kernel's own (streamingt2v_b200/csrc/mtgemm_ring.h, compiled into a small host library);
the four thread roles of mtgemm_alt_kernel -- A/B producer, residual producer, consumer warpgroups 0 and 1 -- are
state machines that follow the kernel's loops.  An mbarrier is modelled as the hardware defines it: a count of completed
phases, a wait on a parity that succeeds when the phase of that parity is the last completed one (so a waiter two
phases ahead passes wrongly), TMA loads that complete asynchronously and in any order.  The two tile counters per
warpgroup that keep a warpgroup from running that far ahead are plain integers.  A seeded random scheduler
interleaves the roles.  Checked: no buffer is refilled before its owner released it, a wait only ever passes on the
fill it was meant for, each warpgroup consumes exactly its own tiles' fills in order, nothing deadlocks and every role
leaves its loop.
"""
import ctypes
import os
import random
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SUB_W = 32

SHIM = r"""
#include "mtgemm_ring.h"
using namespace b200;
extern "C" {
void sim_ring_step(uint32_t* idx, uint32_t* phase, uint32_t depth) { RingPos r{*idx, *phase}; ring_step(r, depth); *idx = r.idx; *phase = r.phase; }
void sim_ring_advance(uint32_t* idx, uint32_t* phase, uint32_t n, uint32_t depth) { RingPos r{*idx, *phase}; ring_advance(r, n, depth); *idx = r.idx; *phase = r.phase; }
uint32_t sim_alt_owner(uint32_t t) { return alt_owner(t); }
uint32_t sim_tile_res_slots(uint32_t n_tile, uint32_t w, uint32_t n_out, uint32_t sub_w, uint32_t nres) { return tile_res_slots(n_tile, w, n_out, sub_w, nres); }
}
"""


@pytest.fixture(scope="module")
def ring(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    d = tmp_path_factory.mktemp("ring")
    src = d / "shim.cpp"
    src.write_text(SHIM)
    so = d / "libring.so"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "streamingt2v_b200", "csrc"), str(src), "-o", str(so)])
    lib = ctypes.CDLL(str(so))
    for f in (lib.sim_alt_owner, lib.sim_tile_res_slots):
        f.restype = ctypes.c_uint32
    return lib


class Pos:
    """RingPos, stepped by the kernel's helpers."""

    def __init__(self, lib, depth):
        self.lib, self.depth = lib, depth
        self.i, self.p = ctypes.c_uint32(0), ctypes.c_uint32(0)

    idx = property(lambda s: s.i.value)
    phase = property(lambda s: s.p.value)

    def step(self):
        self.lib.sim_ring_step(ctypes.byref(self.i), ctypes.byref(self.p), self.depth)

    def advance(self, n):
        self.lib.sim_ring_advance(ctypes.byref(self.i), ctypes.byref(self.p), n, self.depth)


class Ring:
    """`depth` buffers with a full and an empty mbarrier each (one arrival completes a phase), plus the shadow state
    the checks need: which fill a buffer holds, whether it has landed, whether its owner released it."""

    def __init__(self, depth):
        self.depth = depth
        self.full = [0] * depth      # completed phases of the full barrier
        self.empty = [0] * depth     # completed phases of the empty barrier
        self.fill = [None] * depth   # number of the fill issued into the buffer
        self.landed = [False] * depth
        self.released = [True] * depth
        self.issued = 0
        self.inflight = []           # buffers whose TMA load has not completed

    @staticmethod
    def passes(completed, parity):
        """mbarrier.try_wait.parity: true when the phase of that parity is not the one in progress."""
        return (completed & 1) != parity

    def issue(self, b):
        assert self.released[b], f"buffer {b} refilled before fill {self.fill[b]} was released"
        self.fill[b], self.landed[b], self.released[b] = self.issued, False, False
        self.issued += 1
        self.inflight.append(b)

    def land(self, k):
        b = self.inflight.pop(k)
        self.landed[b] = True
        self.full[b] += 1

    def release(self, b):
        self.released[b] = True
        self.empty[b] += 1


def _producer(ring, fills_per_tile):
    """produce_ab / produce_residuals: every fill of every tile in order, waiting on `empty` with parity ph ^ 1."""
    st, ph = 0, 0
    for n in fills_per_tile:
        for _ in range(n):
            while not Ring.passes(ring.empty[st], ph ^ 1):
                yield
            ring.issue(st)
            st += 1
            if st == ring.depth:
                st, ph = 0, ph ^ 1
            yield


def _wait_fill(ring, pos, want, who):
    """A consumer-side wait on the full barrier at `pos`; it must pass on fill number `want` and no other."""
    while not Ring.passes(ring.full[pos.idx], pos.phase):
        yield
    assert ring.fill[pos.idx] == want and ring.landed[pos.idx], \
        f"{who}: wait for fill {want} passed on buffer {pos.idx} holding fill {ring.fill[pos.idx]} " \
        f"(landed={ring.landed[pos.idx]})"


def _consumer(lib, cw, tiles, ipt, res_per_tile, ab, rr, log, done, ordered=True):
    """The consumer loop of mtgemm_alt_kernel for warpgroup `cw`.  done = the shared tile counters [w], [2 + w]."""
    pa = Pos(lib, ab.depth)
    pr = Pos(lib, rr.depth) if rr is not None else None
    a_no = r_no = 0   # number of the fill at the current ring positions
    for t in range(tiles):
        if lib.sim_alt_owner(t) != cw:
            if t + 1 >= tiles:
                break
            pa.advance(ipt)
            if rr is not None:
                pr.advance(res_per_tile[t])
            a_no += ipt
            r_no += res_per_tile[t]
            continue
        while ordered and done[1 - cw] < t:
            yield
        prev = None
        for i in range(ipt):
            yield from _wait_fill(ab, pa, a_no, f"wg{cw} tile {t}")
            if i + 1 == ipt:
                done[cw] = t + 1
            log.append(("ab", t, a_no))
            if prev is not None:
                ab.release(prev)
            prev = pa.idx
            pa.step()
            a_no += 1
            yield
        ab.release(prev)
        while ordered and rr is not None and done[2 + 1 - cw] < t:
            yield
        for _ in range(res_per_tile[t]):   # the epilogue takes the tile's residual slots in order
            yield from _wait_fill(rr, pr, r_no, f"wg{cw} tile {t} residual")
            log.append(("res", t, r_no))
            yield
            rr.release(pr.idx)
            pr.step()
            r_no += 1
        if rr is not None:
            done[2 + cw] = t + 1
        yield


def simulate(lib, *, tiles, ipt, stages, nres, res_slots, n_tiles, tile_out_w, n_out, seed, ordered=True):
    """One CTA with `tiles` tiles.  Returns the per-warpgroup logs; raises AssertionError on a protocol violation."""
    rng = random.Random(seed)
    res_per_tile = [lib.sim_tile_res_slots(t % n_tiles, tile_out_w, n_out, SUB_W, nres) for t in range(tiles)]
    ab = Ring(stages)
    rr = Ring(res_slots) if nres else None
    logs = ([], [])
    done = [0, 0, 0, 0]
    actors = {"prod": _producer(ab, [ipt] * tiles)}
    if rr is not None:
        actors["res"] = _producer(rr, res_per_tile)
    for cw in (0, 1):
        actors[f"wg{cw}"] = _consumer(lib, cw, tiles, ipt, res_per_tile, ab, rr, logs[cw], done, ordered)
    idle = 0
    while actors:
        choices = list(actors) + [("land", r) for r in (ab, rr) if r is not None and r.inflight]
        c = rng.choice(choices)
        before = (ab.full[:], ab.empty[:], ab.issued, rr and (rr.full[:], rr.empty[:], rr.issued), len(actors), done[:])
        if isinstance(c, tuple):
            c[1].land(rng.randrange(len(c[1].inflight)))
        else:
            try:
                next(actors[c])
            except StopIteration:
                del actors[c]
        after = (ab.full[:], ab.empty[:], ab.issued, rr and (rr.full[:], rr.empty[:], rr.issued), len(actors), done[:])
        idle = idle + 1 if before == after and not isinstance(c, tuple) else 0
        assert idle < 2000, f"deadlock: {sorted(actors)} cannot make progress"
    assert not ab.inflight and (rr is None or not rr.inflight), "a load is still in flight after every role left"
    for cw in (0, 1):
        want_ab = [(t, t * ipt + i) for t in range(cw, tiles, 2) for i in range(ipt)]
        assert [(t, f) for k, t, f in logs[cw] if k == "ab"] == want_ab, f"wg{cw} consumed the wrong stages"
        starts = [sum(res_per_tile[:t]) for t in range(tiles)]
        want_res = [(t, starts[t] + i) for t in range(cw, tiles, 2) for i in range(res_per_tile[t])]
        assert [(t, f) for k, t, f in logs[cw] if k == "res"] == want_res, f"wg{cw} consumed the wrong residual slots"
    return logs


# (n_tiles, tile_out_w, n_out): one full N tile; a ragged last N tile of three; GEGLU at bn = 128 (64 outputs a tile)
N_LAYOUTS = [(1, 128, 128), (3, 160, 330), (2, 64, 128)]


@pytest.mark.parametrize("stages", [3, 4, 5, 6])
@pytest.mark.parametrize("nres", [0, 1, 2])
def test_alternating_protocol(ring, stages, nres):
    runs = 0
    for tiles in (0, 1, 2, 3, 4, 7, 10):
        for ipt in (1, 2, 3, stages - 1, stages, stages + 1, 2 * stages + 1, 20):
            for n_tiles, tile_out_w, n_out in N_LAYOUTS:
                want = nres * (tile_out_w // SUB_W)
                for res_slots in sorted({max(nres, 2), want}) if nres else [0]:
                    for seed in range(3):
                        simulate(ring, tiles=tiles, ipt=ipt, stages=stages, nres=nres, res_slots=res_slots,
                                 n_tiles=n_tiles, tile_out_w=tile_out_w, n_out=n_out, seed=seed)
                        runs += 1
    assert runs >= 500


def test_single_tile_leaves_warpgroup_1_nothing_to_wait_for(ring):
    logs = simulate(ring, tiles=1, ipt=5, stages=4, nres=2, res_slots=8, n_tiles=1, tile_out_w=128, n_out=128, seed=0)
    assert logs[1] == []
    g = _consumer(ring, 1, 1, 5, [8], Ring(4), Ring(8), [], [0, 0, 0, 0])
    with pytest.raises(StopIteration):   # leaves its loop at once, although no stage has been filled
        next(g)


def test_simulation_sees_a_wait_two_phases_ahead(ring):
    """Without the tile counters a warpgroup can reach a buffer two phases ahead of its barrier (3 stages, 1 k-block
    a tile: warpgroup 0 goes from fill 2 to fill 4 while fill 1, in the same buffer, is still in flight), and its
    wait passes on the wrong fill.  The simulation must catch that, or it proves nothing about the counters."""
    caught = 0
    for seed in range(300):
        try:
            simulate(ring, tiles=8, ipt=1, stages=3, nres=0, res_slots=0, n_tiles=1, tile_out_w=128, n_out=128,
                     seed=seed, ordered=False)
        except AssertionError:
            caught += 1
    assert caught > 0


def test_ring_advance_is_repeated_steps(ring):
    for depth in (2, 3, 4, 5, 6, 16):
        for start in range(2 * depth):
            for n in (0, 1, depth - 1, depth, depth + 1, 3 * depth + 2, 180):
                a, b = Pos(ring, depth), Pos(ring, depth)
                a.advance(start)
                for _ in range(start):
                    b.step()
                a.advance(n)
                for _ in range(n):
                    b.step()
                assert (a.idx, a.phase) == (b.idx, b.phase)


def test_alternating_kernels_32_64_128_in_the_library():
    """The alternating instantiations are exactly the N tiles 32, 64 and 128 (the 160-wide tile has none), and each
    uses wgmma, TMA loads and TMA stores."""
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    import re
    import __graft_entry__ as g
    g.build()
    from streamingt2v_b200 import _lib
    out = subprocess.run(["cuobjdump", "-sass", str(_lib.lib_path())], capture_output=True, text=True, check=True).stdout
    alt = [b for b in re.split(r"Function : ", out) if "mtgemm_alt_kernel" in b.splitlines()[0]]
    tiles = sorted(int(re.search(r"mtgemm_alt_kernelILi(\d+)E", b.splitlines()[0]).group(1)) for b in alt)
    assert tiles == [32, 64, 128], [b.splitlines()[0] for b in alt]
    for b in alt:
        for needle in ("HGMMA", "UTMALDG", "UTMASTG", "USETMAXREG"):
            assert needle in b, (b.splitlines()[0], needle)


def test_eight_gemm_kernels_do_not_spill(tmp_path):
    """mtgemm.cu compiles to eight GEMM kernels (cooperative N tiles 32, 64, 128, 160, 256; alternating 32, 64, 128)
    and ptxas reports 0 spill bytes for each."""
    import re
    from streamingt2v_b200 import build
    src = os.path.join(ROOT, "streamingt2v_b200", "csrc", "mtgemm.cu")
    r = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "m.o")],
                       capture_output=True, text=True, check=True)
    rows = re.findall(r"Compiling entry function '(\S+)'.*\n.*\n.*?(\d+) bytes spill stores, (\d+) bytes spill loads",
                      r.stderr)
    kernels = sorted(re.search(r"(mtgemm_kernel|mtgemm_alt_kernel)ILi(\d+)E", name).groups() for name, _, _ in rows)
    assert kernels == sorted([("mtgemm_kernel", str(n)) for n in (32, 64, 128, 160, 256)] +
                             [("mtgemm_alt_kernel", str(n)) for n in (32, 64, 128)]), r.stderr
    for name, st, ld in rows:
        assert (st, ld) == ("0", "0"), (name, st, ld)
