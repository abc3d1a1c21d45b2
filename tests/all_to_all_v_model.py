"""Bit-exact model of the all-to-all with variable segments (csrc/allreduce.cu alltoallv_kernel, ``SymmWorld.all_to_all_v_``).
Shared by tests/test_gpu_all_to_all_v_emulated.py and the CPU test tests/test_all_to_all_v_model.py.

* Rank s sends ``sends[s][d]`` (uint8 bytes) to rank d.  Rank r's output buffer holds one segment per source p at byte
  ``out_offsets[r][p]``, ``out_lens[r][p]`` bytes long: what r expects from p.
* The receiver takes min(what was sent, what it expects) bytes of each pair, from the start of the segment; the rest of its
  segment and every byte outside the segments keep what they held, so splits that disagree between ranks truncate.
* The kernel runs max(1, ceil(longest send / chunk)) rounds of one barrier each after the header barrier, on every rank.
* Every function takes what the outputs held before the call and returns them whole after it (sentinels included).
* ``fault`` plants known bugs; tests/test_all_to_all_v_model.py shows the checker catches each.
"""
import torch


def take(sent: int, expected: int, fault: str = None) -> int:
    """Bytes a receiver moves for one pair.  ``fault`` "sent": it trusts the sender's length (writes past a short segment);
    "expected": it trusts its own (reads past a short send)."""
    if fault == "sent":
        return sent
    if fault == "expected":
        return expected
    return min(sent, expected)


def predict(sends: list, out_before: list, out_offsets: list, out_lens: list, fault: str = None) -> list:
    """Every rank's output buffer (uint8, whole) after the call.  ``fault`` also "swap" (rank r receives from source p what
    p sent to r ^ 1), "tail" (the last partial 16-byte vector of each pair is dropped)."""
    world = len(sends)
    outs = [o.clone() for o in out_before]
    for r in range(world):
        for p in range(world):
            src = sends[p][r ^ 1 if fault == "swap" and (r ^ 1) < world else r]
            n = take(src.numel(), out_lens[r][p], fault)
            if fault == "tail":
                n = n // 16 * 16
            if n > src.numel():                  # a planted fault overruns the send: it reads zeros of a fresh staging buffer
                src = torch.cat([src, torch.zeros(n - src.numel(), dtype=torch.uint8)])
            at = out_offsets[r][p]
            outs[r][at:at + n] = src[:n]
    return outs


def rounds(send_lens: list, chunk: int) -> int:
    """The kernel's round count for a W x W matrix of send lengths in bytes (the same on every rank)."""
    longest = max((n for row in send_lens for n in row), default=0)
    return max(1, -(-longest // chunk))


def barriers(send_lens: list, chunk: int) -> int:
    """Barriers of one call: the header barrier and one per round (so the per-block epochs advance by this much)."""
    return 1 + rounds(send_lens, chunk)


def split_offsets(splits: list, row_bytes: int) -> list:
    """Byte offsets of the segments a split list cuts from dim 0, and the end."""
    offs = [0]
    for n in splits:
        offs.append(offs[-1] + n * row_bytes)
    return offs


def single_form(inputs: list, in_splits: list, outputs_before: list, out_splits: list) -> list:
    """``all_to_all_single`` with split sizes on every rank: ``inputs[s]`` / ``outputs_before[r]`` are tensors of one dtype
    whose dim 0 the split lists cut.  Returns every output after the call, through :func:`predict`."""
    world = len(inputs)
    as_u8 = lambda t: t.reshape(-1).view(torch.uint8)  # noqa: E731
    row = lambda t: (t.numel() // t.shape[0] if t.shape[0] else 0) * t.element_size()  # noqa: E731
    sends = []
    for s, x in enumerate(inputs):
        o = split_offsets(in_splits[s], row(x))
        sends.append([as_u8(x)[o[d]:o[d + 1]] for d in range(world)])
    offs, lens = [], []
    for r, y in enumerate(outputs_before):
        o = split_offsets(out_splits[r], row(y))
        offs.append(o[:-1])
        lens.append([o[p + 1] - o[p] for p in range(world)])
    got = predict(sends, [as_u8(y).clone() for y in outputs_before], offs, lens)
    return [g.view(y.dtype).view(y.shape) for g, y in zip(got, outputs_before)]


def by_slicing(inputs: list, in_splits: list) -> list:
    """Plain torch: rank r's output is the concatenation over p of the rows rank p's splits give r (consistent splits)."""
    world = len(inputs)
    outs = []
    for r in range(world):
        parts = []
        for p, x in enumerate(inputs):
            start = sum(in_splits[p][:r])
            parts.append(x[start:start + in_splits[p][r]])
        outs.append(torch.cat(parts))
    return outs
