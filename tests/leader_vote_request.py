"""Leaders for the tests of vote requests at a leader (raftgpu_leader_vote_request_wire,
oracle/leader_vote_request_oracle.c): random leader groups with the caller's voter table, the caller's host side of an
answered frame, and the resubmission loop -- this pass, its host side, the host's step of a COMMIT_VOTE frame, and
raftgpu_vote_request_wire on the frames of the groups that are Followers -- until no frame is left."""
import numpy as np

from helpers import B
from oracle import leader_vote_request_oracle as LV
from oracle import vote_request_oracle as VR
import hb_frames as F
import pass_forms as PF
import vote_request_frames as Q

# the device form in pass_forms' table: raftgpu_vote_request_wire's arguments, outputs and bound
PF.PASSES.setdefault("leader_vote_request_wire", PF._frame_pass(PF.VOTERS, PF.ST + PF.OUT, PF.REPLY,
                                                                B.vote_request_wire_bound))
NAMES = ("status", "out", "bytes", "offsets", "totals")


def scenario(rng, n_narrow, n_wide, p_check_quorum=0.5):
    """Q.Scenario's groups, table and setup with every group a Leader (vote = its own id, RAFTGPU_VOTER_LEADER, in
    lease for half of them); VR.CHECK_QUORUM, the literal form's own bit, on a share of them."""
    s = Q.Scenario(rng, n_narrow, n_wide, p_role=(0.0, 0.0, 0.0, 1.0))
    for g in s.lows:
        if rng.random() < p_check_quorum:
            s.table["flags"][g] |= VR.CHECK_QUORUM
    return s


def group_of(frame) -> int:
    return int(np.frombuffer(frame[:4], "<u4")[0]) >> 4


def host_side(table, role, status, out, frames_):
    """The caller's side of the OK frames of either vote-request pass: Q.caller_update, and the follower selection of
    a group a bump made a Follower."""
    Q.caller_update(table, role, status, out, frames_)
    for i in np.flatnonzero((status >> 4 == B.WIRE_OK) & ((status & B.VREQ_BUMPED) != 0)):
        table["flags"][group_of(frames_[i])] |= B.VOTER_SELECT


def responses(blob, off, into):
    """Append each response to its group's list, in order."""
    for k in range(len(off) - 1):
        fr = blob[off[k]:off[k + 1]].tobytes()
        into.setdefault(group_of(fr), []).append(fr)


def settle(c, q, vt, role, table, frames_, leader_pass, voter_pass):
    """The resubmission loop over frames_ (in frame order) from the state (c, q, vt, role, table), changed in place.
    Each round runs leader_pass (this pass) on the pending frames, then voter_pass (raftgpu_vote_request_wire) on those
    it left ROLE; the host side follows each pass, and the host steps a COMMIT_VOTE frame with the literal form.  The
    DUP frames of both passes are the next round's, in frame order.  Both passes are called as pass(blob, off, table)
    -> (status, out, blob, offsets, totals) -> ({group: [responses]}, rounds, status counts of either pass)."""
    got, pending, rounds, kinds = {}, list(range(len(frames_))), 0, np.zeros((2, 16), np.int64)
    while pending:
        dups = []
        for k, run in enumerate((leader_pass, voter_pass)):
            if not pending:
                break
            fr = [frames_[i] for i in pending]
            st, out, rb, ro, _ = run(*F.batch(fr), table)
            kinds[k] += np.bincount(st >> 4, minlength=16)
            responses(rb, ro, got)
            host_side(table, role, st, out, fr)
            for j in np.flatnonzero(st >> 4 == B.WIRE_COMMIT_VOTE):   # RawNode::step on the host
                responses(*VR.literal(c, q, vt, role, table, *F.batch([fr[j]]))[:2], got)
                table["flags"][group_of(fr[j])] |= B.VOTER_SELECT        # (it leaves a Follower)
            dups += [pending[j] for j in np.flatnonzero(st >> 4 == B.WIRE_DUP)]
            pending = [pending[j] for j in np.flatnonzero(st >> 4 == B.WIRE_ROLE)] if k == 0 else []
        pending = sorted(dups)
        rounds += 1
    return got, rounds, kinds


def oracle_passes(c, q, vt):
    """The batch oracles of this pass and of raftgpu_vote_request_wire over (c, q, vt), as settle takes them."""
    return (lambda blob, off, t: LV.batch(c, q, vt, blob, off, t),
            lambda blob, off, t: VR.batch(c, q, vt, blob, off, t))


def literal(c, q, vt, role, table, frames_):
    """The literal form over frames_ in frame order -> {group: [responses]}."""
    blob, off = F.batch(frames_)
    rb, ro, _ = VR.literal(c, q, vt, role, table, blob, off)
    got = {}
    responses(rb, ro, got)
    return got
