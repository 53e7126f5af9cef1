"""The shapes of test_gpu_exchange_shapes.py reach every kernel instantiation of csrc/exchange.cu.

The CALL_SEND / CALL_RECV ladders and pick_vec's rule are parsed out of the source, so a new rung or a moved
threshold fails here until exchange_cases.SHAPES reaches it again: every sender `<VEC, CHUNKS>` both on its FULL
path and off it, every receiver `<VEC, CHUNKS>`."""
import os
import re

import pytest

from exchange_cases import RECV_VIEWS, SHAPES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "adaqp_b200", "csrc", "exchange.cu")
MAX_F = 1024


def source():
    with open(SRC) as f:
        return f.read()


def function_body(src, name):
    m = re.search(r"\n(?:inline )?int " + name + r"\(", src)
    assert m, f"{name} not found in exchange.cu"
    end = src.index("\n}\n", m.end())
    return src[m.end():end]


def pick_vec_rule(src):
    """Order of the vector widths pick_vec tries; the conditions of its `ok` lambda are checked to be the ones
    modelled by `pick_vec` below."""
    body = function_body(src, "pick_vec")
    for cond in (r"F % vec", r"ld % vec", r"\(uintptr_t\)vec \* 4 - 1", r"\(uintptr_t\)p0 & m"):
        assert re.search(cond, body), f"pick_vec no longer tests `{cond}`: update the model in this file"
    order = [int(v) for v in re.findall(r"if \(ok\((\d)\)\) return \1;", body)]
    order.append(int(re.search(r"\n\s*return (\d);\s*$", body).group(1)))
    assert order[-1] == 1 and sorted(order, reverse=True) == order, order
    return order


def ladders(src, fn, macro):
    """{VEC: [(nchunks bound or None for the final else, CHUNKS)]} of the launcher `fn`."""
    body = function_body(src, fn)
    out, vec = {}, None
    for line in body.splitlines():
        line = line.strip()
        m = re.match(r"(?:\} else )?if \(vec == (\d)\) \{$", line)
        if m:
            vec = int(m.group(1))
            continue
        if line == "} else {":
            vec = 1
            continue
        m = re.match(r"(?:else )?(?:if \(nchunks <= (\d+)\) )?" + macro + r"\((\d), (\d+)\);$", line)
        if m:
            assert vec is not None and int(m.group(2)) == vec, line
            out.setdefault(vec, []).append((int(m.group(1)) if m.group(1) else None, int(m.group(3))))
    assert sorted(out) == [1, 2, 4], out
    for v, rungs in out.items():
        assert rungs[-1][0] is None and all(b is not None for b, _ in rungs[:-1]), (v, rungs)
    return out


def pick_vec(order, F, ld, base_mod16):
    for v in order[:-1]:
        if F % v == 0 and ld % v == 0 and base_mod16 % (4 * v) == 0:
            return v
    return order[-1]


def rung(ladder, vec, F):
    nchunks = (F + 32 * vec - 1) // (32 * vec)
    for bound, chunks in ladder[vec]:
        if bound is None or nchunks <= bound:
            return chunks


@pytest.fixture(scope="module")
def parsed():
    src = source()
    return pick_vec_rule(src), ladders(src, "adaqp_send_quant", "CALL_SEND"), ladders(src, "adaqp_recv_quant", "CALL_RECV")


def test_every_width_fits_its_rung(parsed):
    """Every F the launchers accept lands on a rung wide enough for it, for every vector width."""
    _, send, recv = parsed
    for ladder in (send, recv):
        for vec in ladder:
            for F in range(vec, MAX_F + 1, vec):
                assert 32 * vec * rung(ladder, vec, F) >= F, (vec, F)


def test_shapes_reach_every_sender_instantiation(parsed):
    order, send, _ = parsed
    reached = set()
    for s in SHAPES:
        v = pick_vec(order, s.F, s.ld, s.base_mod16)
        c = rung(send, v, s.F)
        reached.add((v, c, s.F == 32 * v * c))
    want = {(v, c, full) for v, rungs in send.items() for _, c in rungs for full in (False, True)}
    assert reached == want, sorted(want - reached)


def test_shapes_reach_every_receiver_instantiation(parsed):
    order, _, recv = parsed
    reached = set()
    for s in SHAPES:
        # the exchange's own receive writes the halo at a 256-byte aligned slab offset with ld = F
        for pad, col in ((0, 0),) + RECV_VIEWS:
            v = pick_vec(order, s.F, s.F + pad, (4 * col) % 16)
            reached.add((v, rung(recv, v, s.F)))
    want = {(v, c) for v, rungs in recv.items() for _, c in rungs}
    assert reached == want, sorted(want - reached)


def test_strided_receive_views_reach_vec2_and_vec1(parsed):
    """The second receive into RECV_VIEWS is what reaches the receiver's narrow paths at F % 4 == 0."""
    order = parsed[0]
    vecs = [pick_vec(order, 256, 256 + pad, (4 * col) % 16) for pad, col in RECV_VIEWS]
    assert vecs == [2, 1]

