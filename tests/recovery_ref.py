"""A restatement of the stream recovery's decision rule (include/sl2b200.h, sl2_set_stream_recovery; csrc/recover.cu
recover_kernel and the acceptance in reloc_kernel) as a state machine, one stream at a time.

A state is a dict with the fields of sl2_recovery_result that the rule moves: lost, failed_steps, lost_steps,
attempted and recoveries.  A setting is a dict with lost_after, min_matches and retry_period.  `broken` names a
deliberate mistake, so that the tests can show each named check catches one."""

FIELDS = ("lost", "failed_steps", "lost_steps", "attempted", "recoveries")


def fresh():
    """The state the setter leaves: tracking, no counts, no result."""
    return dict.fromkeys(FIELDS, 0)


def reset(st):
    """The resets other than the setter (snapshot load, sl2_set_state, sl2_set_features, an accepted sl2_relocalise):
    back to tracking with zero counts; attempted and recoveries describe the past and stay."""
    return dict(st, lost=0, failed_steps=0, lost_steps=0)


def selects(cfg, st, broken=()):
    """Rule 4: whether the step a stream enters with state st selects features."""
    if "select_while_lost" in broken:
        return True
    if "off_keeps_lost" in broken:
        return not st["lost"]
    return not (cfg["lost_after"] > 0 and st["lost"])


def end_of_step(cfg, st, nmeas, accept, broken=()):
    """Rules 1-3 at the end of a fused step whose record shows nmeas.  accept() performs the try and says whether it
    was accepted.  Returns (the new state, whether the step tried)."""
    st = dict(st)
    if cfg["lost_after"] <= 0:
        return st, False
    tries = False
    if st["lost"]:
        st["lost_steps"] += 1
        if "retry_before_count" in broken:
            tries = (st["lost_steps"] - 1) % cfg["retry_period"] == 0
        else:
            tries = st["lost_steps"] % cfg["retry_period"] == 0
    else:
        fail = nmeas <= cfg["min_matches"] if "fail_at_min" in broken else nmeas < cfg["min_matches"]
        if "failures_accumulate" in broken:
            st["failed_steps"] = st["failed_steps"] + 1 if fail else st["failed_steps"]
        else:
            st["failed_steps"] = st["failed_steps"] + 1 if fail else 0
        declare = st["failed_steps"] > cfg["lost_after"] if "late_declaration" in broken else \
            st["failed_steps"] >= cfg["lost_after"]
        if declare:
            st["lost"], st["lost_steps"] = 1, 0
            tries = "no_try_on_declaration" not in broken
    st["attempted"] = int(tries)
    if tries and accept():
        st["recoveries"] += 1
        st["lost"], st["lost_steps"] = 0, 0
        if "keep_failed_on_accept" not in broken:
            st["failed_steps"] = 0
    return st, tries


def run(cfg, nmeas_seq, accepted=lambda t: False, broken=(), off_at=None):
    """The states after each step of a stream whose steps measure nmeas_seq[t]; a try at step t is accepted when
    accepted(t).  off_at: the step before which the setter turns the feature off (lost_after = 0).  Returns a list of
    (state after step t, tried at t, selected at t)."""
    st, out = fresh(), []
    for t, n in enumerate(nmeas_seq):
        if off_at is not None and t == off_at:
            cfg = dict(cfg, lost_after=0)
            if "off_keeps_lost" not in broken:
                st = fresh()
        sel = selects(cfg, st, broken)
        st, tried = end_of_step(cfg, st, n if sel else 0, lambda: accepted(t), broken)
        out.append((st, tried, sel))
    return out


BROKEN = ("select_while_lost", "off_keeps_lost", "retry_before_count", "fail_at_min", "failures_accumulate",
          "late_declaration", "no_try_on_declaration", "keep_failed_on_accept")
