"""Plain restatements of what vp8gpu_decode_ivf with device-side tokens decides on the host, for the tests of
tools/make_pipeline_stream.py: the token capacity of a frame (Engine::token_cap_for), the arena size of plan() and the
placement of every frame's token piece by arena_take in IvfDecode::worker_device, in the order in which a worker
stages its frames (chunks, slow start, slot reuse).  With one worker the placement does not depend on timing."""
import collections

K_TOK_SLOTS, K_TOK_CHUNK = 96, 32


def token_cap_for(bits, n_mbs):
    """tokens k_tokens may write for `bits` partition bytes: 9 per byte (rounded up to 256 bytes, plus 16) + 1024,
    at most 400 per macroblock"""
    return min(((bits + 16 + 255) // 256 * 256) * 9 + 1024, n_mbs * 400)


def frame_tag(frame):
    """(key frame, shown, first partition bytes, header bytes) of a compressed frame"""
    tag = frame[0] | frame[1] << 8 | frame[2] << 16
    key = not (tag & 1)
    return key, bool(tag >> 4 & 1), tag >> 5 & 0x7FFFF, 10 if key else 3


def partition_bytes(frame, nparts):
    """TokenWork::bits_len: the DCT partitions without their size table"""
    _, _, first, hdr = frame_tag(frame)
    return len(frame) - hdr - first - 3 * (nparts - 1)


def needs_per_gop(frames, nparts, n_mbs):
    """token_cap_for of every frame, per GOP of the items vp8gpu_decode_ivf decodes (from the first key frame on,
    split at key frames); nparts: DCT partitions of every frame"""
    out = []
    for f, p in zip(frames, nparts):
        if len(f) > 0 and not (f[0] & 1):
            out.append([])
        if out:
            out[-1].append(token_cap_for(partition_bytes(f, p), n_mbs))
    return out


def plan(slots, max_frame_bytes, n_mbs, chunk=None, arena=None):
    """(tok_slots, tok_chunk, arena tokens, worst) of one worker on a device with memory to spare; chunk / arena:
    VP8GPU_TOK_CHUNK / VP8GPU_TOK_ARENA (None = not set)"""
    worst = token_cap_for(max_frame_bytes, n_mbs)
    tok_chunk = min(slots // 3, K_TOK_CHUNK) if slots // 3 > 0 else 1
    if chunk is not None and 1 <= chunk <= slots // 2:
        tok_chunk = chunk
    floor = (slots // 2 + 2) * worst
    cap = max(slots * worst, floor) if arena is None else max(arena * worst, floor)
    return slots, tok_chunk, cap, worst


class ArenaTooSmall(Exception):
    pass


def simulate(needs, slots, chunk, cap):
    """arena_take over one worker's frames: needs = per GOP, the token capacity of every frame.
    -> Counter(takes, wraps, waits) as VP8GPU_TRACE prints them"""
    n = collections.Counter(takes=0, wraps=0, waits=0)
    live = collections.deque()   # slots holding arena space, oldest first
    start, held = {}, set()
    head = 0
    launches, next_slot = 0, 0

    def take(si, need, in_chunk):
        nonlocal head
        if si in held:   # the slot's previous frame is done
            live.remove(si)
            held.discard(si)
        while True:
            at = None
            if not live:
                at = 0 if need <= cap else None
            else:
                tail = start[live[0]]
                if head > tail:
                    if cap - head >= need:
                        at = head
                    elif tail >= need:
                        at = 0
                elif tail - head >= need:
                    at = head
            if at is not None:
                n["takes"] += 1
                if at == 0 and head > 0:
                    n["wraps"] += 1
                start[si] = at
                head = at + need
                held.add(si)
                live.append(si)
                return
            if not live or in_chunk(live[0]):
                raise ArenaTooSmall()
            n["waits"] += 1
            held.discard(live.popleft())

    for gop in needs:
        i = 0
        while i < len(gop):
            want = chunk
            if launches < 3 and (2 << launches) < want:
                want = 2 << launches
            launches += 1
            count = min(len(gop) - i, want)
            first = next_slot
            for c in range(count):
                take((first + c) % slots, gop[i + c], lambda s, c=c: (s - first) % slots < c)
            next_slot = (first + count) % slots
            i += count
    return n
