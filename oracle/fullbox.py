"""Host restatement of the full-box probe's schedule (cro_probe_all), from the rules include/croprobe.h states at
cro_selftest_p2p_plan and DESIGN.md §5: the 1-factorisation rounds, the one prefix every leg moves, which pairs are
scheduled and which peers each device's verdict checks, the ordered stream operations, and a small event-graph
simulator that answers "does X happen before Y".  It also builds the slots a healthy box leaves behind, for
oracle/verdict.py's p2p_finalize.

Pure Python; nothing here imports the product.  An op is a tuple (kind, dev, peer, event, round, slot, bytes), the
fields of cro_p2p_op in order.
"""
from __future__ import annotations

from typing import Callable, Dict, List, NamedTuple, Optional, Sequence, Tuple

import verdict as V

MAX_DEVICES = 16
ACCESS_COLUMNS = 8                 # cro_probe_result.p2p_access has 8 entries
F_SKIP_P2P, F_SKIP_P2P_WRITE = 0x0002, 0x0080
COPY_TMA_FUSED = 3
OP_HBM, OP_PREFIX, OP_RECORD, OP_WAIT, OP_READ, OP_PUSH, OP_REREAD, OP_CHASE, OP_FINALIZE = range(1, 10)
EV_HBM, EV_PUSH, EV_REREAD, EV_CHASE = range(1, 5)
LEGS = (OP_READ, OP_PUSH, OP_REREAD)


class Op(NamedTuple):
    kind: int
    dev: int
    peer: int
    event: int = 0
    round: int = 0
    slot: int = 0
    bytes: int = 0


class Fin(NamedTuple):
    n: int = 0
    self: int = 0
    have_push: int = 0
    push_folded: int = 0
    p2p_bytes: int = 0
    peer_mask: int = 0
    chase_mask: int = 0


class Plan(NamedTuple):
    p2p_bytes: int
    rounds: List[List[Tuple[int, int]]]
    ops: List[Op]
    fin: List[Fin]                 # MAX_DEVICES entries; all zero for a device without a finalize


def rounds_of(n: int) -> List[List[Tuple[int, int]]]:
    """The round-robin 1-factorisation of K_m, m = n rounded up to even: round r holds (m-1, r), then
    ((r+k) mod (m-1), (r-k) mod (m-1)) for k = 1 .. m/2 - 1; a pair with the bye vertex m-1 of an odd n is dropped."""
    if n < 2:
        return []
    m = n + (n % 2)
    out = []
    for r in range(m - 1):
        cand = [(m - 1, r)] + [((r + k) % (m - 1), (r - k) % (m - 1)) for k in range(1, m // 2)]
        out.append([(a, b) for a, b in cand if a < n and b < n])
    return out


def linked(access: Sequence[Sequence[int]], a: int, b: int) -> bool:
    """A pair is scheduled only when both devices have an access column for the other and both directions reach."""
    return a < ACCESS_COLUMNS and b < ACCESS_COLUMNS and bool(access[a][b]) and bool(access[b][a])


def prefix_bytes(sweep_bytes: Sequence[int], p2p_bytes: int) -> int:
    """The one prefix of a call: min(p2p_bytes, every device's S)."""
    return min([p2p_bytes] + list(sweep_bytes))


def checked_peers(n: int, access, unidir: bool) -> List[int]:
    """Per device, the bit mask of peers its verdict checks."""
    rounds = rounds_of(n)
    masks = []
    for i in range(n):
        m = sum(1 << j for j in range(n) if j != i and linked(access, i, j))
        if unidir:                 # the second device of a pair only receives, and checks nothing of the first
            m &= ~sum(1 << a for rd in rounds for a, b in rd if b == i)
        masks.append(m)
    return masks


def plan(sweep_bytes: Sequence[int], p2p_bytes: int, access, flags: int = 0, unidir: bool = False,
         write_variant: int = COPY_TMA_FUSED) -> Plan:
    n = len(sweep_bytes)
    nvlink = n > 1 and not flags & F_SKIP_P2P
    push = nvlink and not flags & F_SKIP_P2P_WRITE
    fin = [Fin()] * MAX_DEVICES
    ops: List[Op] = []
    P = prefix_bytes(sweep_bytes, p2p_bytes) if nvlink else 0
    for i in range(n):
        ops.append(Op(OP_HBM, i, i))
        if nvlink:
            ops += [Op(OP_PREFIX, i, i, slot=V.SLOT_PREFIX, bytes=P), Op(OP_RECORD, i, i, EV_HBM)]
    if not nvlink:
        return Plan(0, [], ops, fin)
    rounds = rounds_of(n)
    for r, rd in enumerate(rounds):
        directed = []
        for a, b in rd:
            if linked(access, a, b):
                directed += [(a, b)] if unidir else [(a, b), (b, a)]
        for a, b in directed:
            ops.append(Op(OP_WAIT, a, b, EV_HBM))
            if r:
                ops.append(Op(OP_WAIT, a, b, EV_REREAD, r - 1))
            ops.append(Op(OP_READ, a, b, 0, r, V.SLOT_P2P0 + 3 * b, P))
            if push:
                ops.append(Op(OP_PUSH, a, b, 0, r, V.SLOT_P2P0 + 3 * b + 1, P))
        ops += [Op(OP_RECORD, i, i, EV_PUSH, r) for i in range(n)]
        for a, b in directed if push else []:
            ops += [Op(OP_WAIT, b, a, EV_PUSH, r), Op(OP_REREAD, b, a, 0, r, V.SLOT_P2P0 + 3 * a + 2, P)]
        ops += [Op(OP_RECORD, i, i, EV_REREAD, r) for i in range(n)]
    ops += [Op(OP_RECORD, i, i, EV_CHASE) for i in range(n)]
    checked = checked_peers(n, access, unidir)
    for i in range(n):
        ops += [Op(OP_WAIT, i, j, EV_CHASE) for j in range(n) if j != i]
        ops += [Op(OP_CHASE, i, i), Op(OP_FINALIZE, i, i)]
        chase = sum(1 << j for j in range(n) if j != i and linked(access, i, j))
        fin[i] = Fin(n, i, int(push and not unidir), int(write_variant == COPY_TMA_FUSED), P, checked[i], chase)
    return Plan(P, rounds, ops, fin)


# ---- the event graph ---------------------------------------------------------------------------------------------------
class Graph:
    """The ops as the GPUs order them: each device's stream runs its ops in order, and a wait orders its stream after
    the last record of that event enqueued before the wait.  A wait with no such record is unbound: it waits on
    whatever an earlier call left in the event, or on nothing."""

    def __init__(self, ops: Sequence[Op]) -> None:
        self.ops = list(ops)
        self.unbound: List[int] = []
        self.before: List[int] = []          # bit k of before[i]: op k happens before op i (or k == i)
        last_on: Dict[int, int] = {}
        last_record: Dict[Tuple[int, int, int], int] = {}
        for i, o in enumerate(self.ops):
            anc = 1 << i
            if o.dev in last_on:
                anc |= self.before[last_on[o.dev]]
            if o.kind == OP_WAIT:
                rec = last_record.get((o.peer, o.event, o.round))
                if rec is None:
                    self.unbound.append(i)
                else:
                    anc |= self.before[rec]
            if o.kind == OP_RECORD:
                last_record[(o.dev, o.event, o.round)] = i
            self.before.append(anc)
            last_on[o.dev] = i

    def happens_before(self, x: int, y: int) -> bool:
        return x != y and bool(self.before[y] >> x & 1)

    def find(self, pred: Callable[[Op], bool]) -> List[int]:
        return [i for i, o in enumerate(self.ops) if pred(o)]


# ---- the healthy box ---------------------------------------------------------------------------------------------------
def healthy_slots(p: Plan, seeds: Sequence[int], nonces: Sequence[int], fold: Callable[[int, int], Tuple[int, int, int]],
                  chase_expect: Sequence[Sequence[int]], t: int = 1000) -> Tuple[List[List[V.Slot]], List[List[int]]]:
    """The slot arrays and chase outputs of every device after a clean call of plan p: fold(seed, words) is the closed
    form of the first `words` words of the pattern of seed.  Device i's pattern is seeds[i]; what it reads of j, and
    what j pushed into its half B, are j's pattern; its own push folds its own pattern (plain copies fold nothing).
    Slots the plan does not write stay armed, and so do the chase rows it does not walk."""
    n = len(seeds)
    slots = [[V.ARMED] * V.SLOT_COUNT for _ in range(n)]
    chase = [[V.MASK64] * (2 * V.MAX_DEVICES) for _ in range(n)]
    for k, o in enumerate(p.ops):
        words = o.bytes // 8
        src = {OP_PREFIX: o.dev, OP_READ: o.peer, OP_PUSH: o.dev, OP_REREAD: o.peer}.get(o.kind)
        if src is not None:
            f = fold(seeds[src], words)
            if o.kind == OP_PUSH and not p.fin[o.dev].push_folded:
                f = (0, 0, 0)
            slots[o.dev][o.slot] = V.Slot(*f, t + k, t + k + 100, nonces[o.dev], words, 0)
        elif o.kind == OP_CHASE:
            for j in range(n):
                if p.fin[o.dev].chase_mask >> j & 1:
                    chase[o.dev][2 * j], chase[o.dev][2 * j + 1] = chase_expect[o.dev][j], 700 + j
    return slots, chase


def finalize_inputs(p: Plan, i: int, slots, chase, chase_expect, nonces, access, hops: int, result: bytes) -> dict:
    """oracle/verdict.py p2p_finalize's arguments for device i of plan p; `result` is what probe_finalize left, whose
    p2p_access becomes device i's access row."""
    f = p.fin[i]
    r = V.Result(result)
    r.set("p2p_access", [int(bool(access[i][j])) if j != i else 0 for j in range(ACCESS_COLUMNS)])
    n = len(nonces)
    return dict(result=r.bytes(), slots=slots[i],
                peer_slots=[slots[j] if j < n and f.peer_mask >> j & 1 else None for j in range(V.MAX_DEVICES)],
                peer_stamp=[nonces[j] if j < n else 0 for j in range(V.MAX_DEVICES)], chase_out=chase[i],
                chase_expect=list(chase_expect[i]) + [0] * (V.MAX_DEVICES - len(chase_expect[i])), n=f.n, self_index=f.self,
                hops=hops, have_push=bool(f.have_push), push_folded=bool(f.push_folded), p2p_bytes=f.p2p_bytes,
                stamp=nonces[i])


def expected_fail(leg: int, push_folded: bool) -> Optional[int]:
    """The fail code a corrupted leg of peer j gives on the device that checks it."""
    return {OP_READ: V.FAIL_P2P_READ, OP_REREAD: V.FAIL_P2P_PUSH, OP_CHASE: V.FAIL_P2P_CHASE,
            OP_PREFIX: V.FAIL_EXPECT, OP_PUSH: V.FAIL_P2P_PUSH if push_folded else None}[leg]
