"""The reference encoder's B-frame coding order and reference-buffer rotation, as host logic over integers.

A resident B-frame sequence needs, for every coded frame, the pictures it reads and the buffer its reconstruction
goes to.  The reference decides this in three places, restated here:
  - the input queue (od_input_queue_batch / od_input_queue_next, reference src/encode.c:289-365): groups of
    b_frames + 1 display frames coded last-first, the last one P (I when the keyframe interval ends there) and the
    others B in display order; a shorter last group at the end of the stream;
  - the golden rule (src/encode.c:2981-2984): keyframes, and every I / P frame whose count of earlier I / P frames is a
    multiple of OD_GOLDEN_FRAME_INTERVAL / (b_frames + 1), never a B frame;
  - the rotation of ref_imgi[GOLD / PREV / NEXT / SELF] over four buffers (src/encode.c:2986-3001 before the frame,
    :3144-3172 after it): with B frames a P frame first moves NEXT into PREV; SELF is the lowest buffer none of
    GOLD / PREV / NEXT holds; afterwards a golden frame becomes GOLD and an I / P frame becomes NEXT (the first one,
    with nothing before it, PREV as well) while PREV takes the old NEXT.  A B frame is never a reference.
The encoder runs with OD_CLOSED_GOP = 0 and without rate control dropping frames (a dropped frame keeps the same
rotation).  The buffer indices serve directly as pool slots of a device-resident sequence: sequence s uses slots
4*s .. 4*s + 3.

pipelined_steps groups one sequence's coded frames into engine steps, so that one sequence fills a batch (new
scheduling, not the reference's): each step holds the next I / P anchor and the B frames coded just before it, which
depend only on pictures finished in earlier steps.  The frames of such a step differ in type, so their quantizers differ
too: the engine takes one quantizer record per frame (config.frame_quant).  With keyframes_inline an I frame joins
such a step too, on an engine with config.frame_types that codes keyframes and P / B frames in one batch.
"""
from collections import namedtuple

I_FRAME, P_FRAME, B_FRAME = 0, 1, 2          # OD_I_FRAME, OD_P_FRAME, OD_B_FRAME (src/state.h:65-67)
GOLD, PREV, NEXT, SELF = 0, 1, 2, 3          # OD_FRAME_* (src/state.h:54-60)
GOLDEN_FRAME_INTERVAL = 10                   # OD_GOLDEN_FRAME_INTERVAL (src/encint.h:76)
MAX_REORDER = 16                             # OD_MAX_REORDER: b_frames <= 15

# One coded frame.  refs: ref_imgi[GOLD, PREV, NEXT, SELF] while the frame is coded (-1: no picture yet); kept: its
# reconstruction (buffer refs[SELF]) is a reference picture afterwards, which is every frame but a B frame.
Frame = namedtuple("Frame", "number type golden refs kept")


def coding_order(nframes, b_frames, keyframe_rate=256):
    """The coded frames of a stream of `nframes` display frames, in coding order (one per daala_encode_packet_out,
    the caller draining the queue after every daala_encode_img_in)."""
    if not 0 <= b_frames < MAX_REORDER or keyframe_rate < 1 or nframes < 0:
        raise ValueError("b_frames is 0..%d and keyframe_rate >= 1" % (MAX_REORDER - 1))
    delay = b_frames + 1
    # the input queue: frames waiting, frames batched for coding, frames since the last keyframe
    input_size, input_head, last_keyframe = 0, 0, keyframe_rate - 1
    queue = []

    def batch(frames):
        nonlocal input_head, input_size, last_keyframe
        kind = P_FRAME
        if last_keyframe + frames == keyframe_rate:
            kind, last_keyframe = I_FRAME, -frames
        queue.append((input_head + frames - 1, kind))                        # the last frame first
        queue.extend((input_head + i, B_FRAME) for i in range(frames - 1))   # then the others in display order
        last_keyframe += frames
        input_head += frames
        input_size -= frames

    def next_frame(end):
        if not queue and input_size > 0:
            next_key = max(keyframe_rate - last_keyframe, 1)
            if input_size >= next_key:
                batch(min(next_key, delay))
            elif input_size >= delay:
                batch(delay)
            elif end:
                batch(min(input_size, delay))
        return queue.pop(0) if queue else None

    order = []
    for i in range(nframes):
        input_size += 1
        while True:
            fr = next_frame(i + 1 == nframes)
            if fr is None:
                break
            order.append(fr)
    # the rotation of the four reference buffers along the coding order
    refi = [-1, -1, -1, -1]
    ip_count = 0
    out = []
    for number, kind in order:
        golden = kind == I_FRAME or (ip_count % (GOLDEN_FRAME_INTERVAL // delay) == 0 and kind != B_FRAME)
        if b_frames and kind == P_FRAME:
            refi[PREV] = refi[NEXT]
        refi[SELF] = min(k for k in range(4) if k not in refi[:SELF])
        out.append(Frame(number, kind, golden, tuple(refi), kind != B_FRAME))
        if golden:
            refi[GOLD] = refi[SELF]
        if not b_frames:
            refi[PREV] = refi[SELF]
        elif kind != B_FRAME:
            if refi[PREV] < 0 and refi[NEXT] < 0:
                refi[PREV] = refi[NEXT] = refi[SELF]
            else:
                refi[PREV], refi[NEXT] = refi[NEXT], refi[SELF]
        if kind != B_FRAME:
            ip_count += 1
    return out


def pipelined_steps(frames, keyframes_inline=False):
    """The coded frames of coding_order(...) as engine steps, in the order they run: [[Frame, ...], ...].

    A P frame forms a step with the B frames coded just before it (the B frames between the two anchors before it),
    all of which read only pictures that earlier steps finished.  An I frame is a step of its own (the keyframe engine,
    whose picture the P-frame engine's pool takes with pool_load); the B frames coded before it form a step of their
    own ahead of it, and so do B frames left at the end of the stream.  Inside a step every frame reads the pool before
    any frame's reconstruction is stored, which is what lets an anchor's SELF buffer be one that the step's B frames
    still read.  The I frames of several sequences may share one step of a keyframe engine with keyframe_quant = 1, each
    at its own record; pool_load from that engine's reconstruction seeds each sequence's P engine as it does for a
    keyframe coded alone.

    keyframes_inline=True: an I frame forms a step with the B frames coded just before it, exactly as a P frame does;
    the steps are those of an engine with frame_types = 1, which codes the keyframe beside them and stores it in the
    pool with ref_slot_out like any other frame."""
    steps, pending = [], []
    for fr in frames:
        if fr.type == B_FRAME:
            pending.append(fr)
        elif fr.type == I_FRAME and not keyframes_inline:
            if pending:
                steps.append(pending)
            steps.append([fr])
            pending = []
        else:
            steps.append([fr] + pending)
            pending = []
    if pending:
        steps.append(pending)
    return steps


def pool_slots(fr, base=0):
    """The pool slots (GOLD, PREV, NEXT) an mc_next engine reads frame `fr` from, its sequence's buffers starting at
    slot `base`.  A frame without a NEXT picture (every frame when b_frames = 0, and I / P frames, which never predict
    from NEXT) names its PREV slot there."""
    gold, prev, nxt = fr.refs[GOLD], fr.refs[PREV], fr.refs[NEXT]
    return base + gold, base + prev, base + (nxt if nxt >= 0 and fr.type == B_FRAME else prev)
