"""The point-to-point layouts of b200mpi.cu restated without a GPU: which layout do_send posts a message
in, how do_recv pulls it, what each side stages in its heap and how many kernels each side launches.
test_p2p_cpu.py pins these rules to the lines of the library they restate; _p2p_worker.py checks every
call's launch count against them on the GPU, which shows that the planned layout is the one that ran.

Sender layouts (do_send):
  direct        a Send from the heap, or an empty message: the receiver pulls from the caller's buffer
  whole/bounce  a host slice of at most kP2PBounceBytes with p2p_fast on, Send or Isend: one copy kernel
                and flag_kernel move it through a mapped pinned bounce into one staging block
  whole/memcpy  an Isend of any other host slice: one cudaMemcpyAsync into one staging block
  whole/kernel  an Isend of device memory: one copy kernel into one staging block
  ring/memcpy   a Send of any other host slice: chunks through up to 4 regions, cudaMemcpyAsync each
  ring/kernel   a Send of device memory outside the heap: chunks through up to 4 regions, a kernel each
Receiver layouts (do_recv):
  none          an empty message
  bounce        a host slice, p2p_fast on, the whole message in its regions and at most kP2PBounceBytes:
                one copy kernel and flag_kernel into a mapped pinned bounce
  device        device memory: one copy kernel per posted chunk, straight into the buffer
  staged        any other host slice: units of at most this rank's stage_chunk, never across the end of
                a posted chunk, each a copy kernel into a heap staging block and a D2H copy
  staged-split  as staged, where a chunk is larger than the unit (several units per chunk)"""
from dataclasses import dataclass

KB, MB = 1 << 10, 1 << 20
BOUNCE_BYTES = 4 * MB     # Ctx::kP2PBounceBytes
MSG_REGIONS = 4           # kMsgRegions
SLOTS_PER_PAIR = 16       # kSlotsPerPair
BOUNCES = 4               # Ctx::kP2PBounces
STAGE_CHUNK = 32 * MB     # Ctx::stage_chunk's default
HOST_MIN_CHUNK = 64 * KB
HEAP_ALIGN = 512          # Heap::alloc rounds every block up to this

SEND_LAYOUTS = ("direct", "whole/bounce", "whole/memcpy", "whole/kernel", "ring/memcpy", "ring/kernel")
RECV_LAYOUTS = ("none", "bounce", "device", "staged", "staged-split")
# Storage of a guarded buffer in the GPU tests: (memory kind, inside this rank's heap)
STORAGES = {"heap": ("device", True), "heap+mis": ("device", True), "torch": ("device", False), "torch+mis": ("device", False),
            "pinned": ("host", False), "torchpin": ("host", False), "pageable": ("host", False)}


def p2p_chunk(nbytes, host, stage_chunk):
    """p2p_chunk(): host slices in chunks of a quarter of the message, 64 KiB to stage_chunk, rounded up
    to 4 KiB; device memory in stage_chunk."""
    if host:
        return min(stage_chunk, max(HOST_MIN_CHUNK, (nbytes // 4 + 4095) // 4096 * 4096))
    return stage_chunk


@dataclass(frozen=True)
class SendPlan:
    layout: str
    chunk: int
    nchunks: int
    nreg: int
    stage: int      # bytes staged in the sender's heap (before Heap::alloc's rounding)
    launches: int


@dataclass(frozen=True)
class RecvPlan:
    layout: str
    unit: int
    units: int
    stage: int      # bytes staged in the receiver's heap
    launches: int


def plan_send(nbytes, host, in_heap, isend, fast, stage_chunk, bounce_free=True):
    """do_send's layout.  bounce_free: whether acquire_bounce finds one of the BOUNCES mapped bounces
    free (all four may be held by other calls of this rank: the message then takes the memcpy form)."""
    direct = nbytes == 0 or (not isend and not host and in_heap)
    bounce = not direct and host and fast and nbytes <= BOUNCE_BYTES and bounce_free
    chunk = nbytes if direct or bounce or isend else min(nbytes, p2p_chunk(nbytes, host, stage_chunk))
    nchunks = 0 if direct else -(-nbytes // chunk)
    nreg = min(max(nchunks, 1), MSG_REGIONS)
    if direct:
        return SendPlan("direct", chunk, 0, nreg, 0, 0)
    fill = "bounce" if bounce else "memcpy" if host else "kernel"
    layout = ("whole/" if bounce or isend else "ring/") + fill
    launches = 2 if bounce else 0 if host else nchunks
    return SendPlan(layout, chunk, nchunks, nreg, chunk * nreg, launches)


def pull_units(nbytes, chunk, unit):
    """[(lo, len)] of the pulls: unit-sized pieces of every chunk, none crossing a chunk's end."""
    out, lo = [], 0
    while lo < nbytes:
        n = min(unit, chunk - lo % chunk, nbytes - lo)
        out.append((lo, n))
        lo += n
    return out


def plan_recv(sp, nbytes, host, fast, stage_chunk, bounce_free=True):
    """do_recv's layout for a message posted as `sp` (plan_send's result)."""
    if nbytes == 0:
        return RecvPlan("none", 0, 0, 0, 0)
    if host and fast and sp.chunk * sp.nreg >= nbytes and nbytes <= BOUNCE_BYTES and bounce_free:
        return RecvPlan("bounce", nbytes, 1, 0, 2)
    unit = min(sp.chunk, stage_chunk) if host else sp.chunk
    units = len(pull_units(nbytes, sp.chunk, unit))
    if not host:
        return RecvPlan("device", unit, units, 0, units)
    return RecvPlan("staged-split" if unit < sp.chunk else "staged", unit, units, unit, units)


@dataclass(frozen=True)
class Case:
    """One message of the matrix: sender and receiver storage, Send or Isend, each side's p2p_fast,
    both sides' stage_chunk, element type and count."""
    send: str
    recv: str
    isend: bool
    send_fast: bool
    recv_fast: bool
    dtype: str
    count: int
    stage_chunk: int = 256 * KB
    recv_stage_chunk: int = 0  # 0: stage_chunk

    @property
    def es(self):
        return ESIZE[self.dtype]

    @property
    def nbytes(self):
        return self.count * self.es

    def plans(self):
        sh, sin = STORAGES[self.send]
        rh, _ = STORAGES[self.recv]
        sp = plan_send(self.nbytes, sh == "host", sin, self.isend, self.send_fast, self.stage_chunk)
        rp = plan_recv(sp, self.nbytes, rh == "host", self.recv_fast, self.recv_stage_chunk or self.stage_chunk)
        return sp, rp

    def pair(self):
        sp, rp = self.plans()
        return sp.layout, rp.layout


ESIZE = {"u8": 1, "f32": 4, "f64": 8, "i64": 8}
DTYPES = ("u8", "f32", "f64", "i64")


def boundaries(stage_chunk=256 * KB):
    """{name: bytes} of every layout rule's edge at this stage_chunk."""
    return {
        "one host chunk": HOST_MIN_CHUNK,                  # a host ring of 1 chunk below, 2 above
        "quarter crosses 64 KiB": 4 * HOST_MIN_CHUNK + 4,  # bytes/4 passes 64 KiB: host chunks grow
        "one device chunk": stage_chunk,                   # a device ring of 1 chunk below, 2 above
        "ring wraps": MSG_REGIONS * stage_chunk,           # 4 regions hold the message below, wrap above;
                                                           # the receiver's bounce condition chunk * nreg >= bytes
        "bounce": BOUNCE_BYTES,                            # kP2PBounceBytes
    }


def boundary_counts(dtype, stage_chunk=256 * KB):
    """0 (a NULL buffer), then one element either side of every boundary, ascending."""
    es = ESIZE[dtype]
    out = {0}
    for b in boundaries(stage_chunk).values():
        out.update((b // es - 1, b // es + 1))
    return sorted(out)


def matrix(world=2, src=0, dst=1, stride=1):
    """The cases of the layout matrix: every sender storage against every receiver storage, Send and
    Isend, p2p_fast {on, off} on each side; the boundary counts and the dtypes rotate as a Latin square
    (the count index and the dtype index walk the cases with coprime steps).  In a world of 2 the
    direction alternates; stride > 1 keeps every stride-th case (a reduced matrix)."""
    out = []
    i = 0
    names = list(STORAGES)
    for si, s in enumerate(names):
        for ri, r in enumerate(names):
            for isend in (False, True):
                for fast in ((True, True), (True, False), (False, True), (False, False)):
                    dt = DTYPES[(si + 3 * ri + isend) % 4]
                    counts = boundary_counts(dt)
                    c = counts[(3 * i + 2 * si + 2 * ri) % len(counts)]
                    if i % stride == 0:
                        a, b = (src, dst) if world > 2 or i % 2 == 0 else (dst, src)
                        out.append((a, b, Case(s, r, isend, fast[0], fast[1], dt, c)))
                    i += 1
    return out


def big_cases():
    """At the default 32 MiB chunk: a pageable Send over 128 MiB (a ring of 32 MiB chunks that wraps)
    and a heap Send of the same size (direct, one chunk) into host receivers, which pull 32 MiB units;
    then rings whose chunks are larger than the receiver's 1 MiB stage_chunk."""
    c = (160 * MB + 4) // 4
    return [Case("pageable", "pageable", False, True, True, "f32", c, STAGE_CHUNK),
            Case("heap", "pageable", False, True, True, "f32", c, STAGE_CHUNK),
            Case("torch", "pinned", False, True, True, "f32", c, STAGE_CHUNK),
            Case("torch+mis", "pageable", False, True, True, "u8", 40 * MB + 3, STAGE_CHUNK, MB),
            Case("pageable", "pinned", False, False, True, "i64", (40 * MB + 8) // 8, STAGE_CHUNK, MB)]


def all_pairs():
    """Every (sender layout, receiver layout) the matrix and big_cases reach."""
    return sorted({c.pair() for _, _, c in matrix()} | {c.pair() for c in big_cases()})


def heap_blocks(nbytes):
    """What Heap::alloc takes for a request of nbytes."""
    return (max(nbytes, 1) + HEAP_ALIGN - 1) // HEAP_ALIGN * HEAP_ALIGN
