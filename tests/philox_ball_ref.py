"""Test-only numpy restatement of the start / goal search's offset stream (art_planner_b200/csrc/artp_sampler.cuh,
ball_offset): Philox4x32-10 with key = seed, counter = (draw lo, draw hi, query, "ARTB"); the two doubles of the block are
taken as in the sampler's stream, offset = r * sqrt(u1) * (cos 2 pi u0, sin 2 pi u0)."""
import numpy as np

from philox_ref import philox4x32_10

TAG = 0x41525442


def ball_words(seed: int, first_draw: int, n: int, n_iter: int) -> np.ndarray:
    """[n, n_iter, 4] uint32 Philox output words of draws first_draw .. first_draw + n_iter - 1 of queries 0 .. n-1."""
    draw = (np.uint64(first_draw) + np.arange(n_iter, dtype=np.uint64))[None, :].repeat(n, 0).reshape(-1)
    q = np.arange(n, dtype=np.uint32)[:, None].repeat(n_iter, 1).reshape(-1)
    ctr = np.stack([(draw & np.uint64(0xFFFFFFFF)).astype(np.uint32), (draw >> np.uint64(32)).astype(np.uint32), q,
                    np.full(draw.shape[0], TAG, np.uint32)], axis=1)
    return philox4x32_10(ctr, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)).reshape(n, n_iter, 4)


def ball_offsets(seed: int, first_draw: int, n: int, n_iter: int, radius) -> np.ndarray:
    """[n, n_iter, 2] offsets; radius scalar or [n]."""
    w = ball_words(seed, first_draw, n, n_iter).astype(np.uint64)
    u0 = ((w[..., 1] << np.uint64(32) | w[..., 0]) >> np.uint64(11)).astype(np.float64) / 9007199254740992.0
    u1 = ((w[..., 3] << np.uint64(32) | w[..., 2]) >> np.uint64(11)).astype(np.float64) / 9007199254740992.0
    r = np.broadcast_to(np.asarray(radius, dtype=np.float64), (n,))[:, None]
    rr = r * np.sqrt(u1)
    a = 2.0 * np.pi * u0
    return np.stack([rr * np.cos(a), rr * np.sin(a)], axis=-1)
