"""A stand-in for VSR.tla in the tests: a `MODULE VSR` with the spec's 20 VARIABLES, the 19 disjunct names of its Next and
every definition the loader looks for, but bodies that are not the spec's.  It has the shape the loader checks
(csrc/vsr_host.cpp, verify_tla) and never the text it verifies, so it loads only as an unverified spec."""

VARIABLES = ["replicas", "rep_status", "rep_log", "rep_view_number", "rep_op_number", "rep_commit_number", "rep_peer_op_number",
             "rep_client_table", "rep_last_normal_view", "rep_svc_recv", "rep_dvc_recv", "rep_sent_dvc", "rep_sent_sv",
             "rep_rec_number", "rep_rec_recv", "clients", "messages", "aux_svc", "aux_restart", "aux_client_acked"]


def module_text(action_names):
    """action_names: the 19 disjuncts of Next in the spec's order"""
    lines = ["------------------------------ MODULE VSR ------------------------------", "EXTENDS Naturals", "",
             "VARIABLES " + ", ".join(VARIABLES), "",
             "Init == replicas = {}", "", "view == replicas", "", "symmValues == {}", ""]
    for inv in ("AcknowledgedWriteNotLost", "AcknowledgedWritesExistOnMajority", "NoLogDivergence", "TestInv"):
        lines += [inv + " == TRUE", ""]
    for a in action_names:
        lines += [a + " ==", "    /\\ replicas' = replicas", "    /\\ UNCHANGED <<rep_status>>", ""]
    lines += ["Next ==", *["    \\/ " + a for a in action_names], "", "===="]
    return "\n".join(lines) + "\n"


def location(text, action):
    """where TLC (and the loader) locate an action of module_text: the extent of its definition's body"""
    lines = text.split("\n")
    i = lines.index(action + " ==")
    return "line %d, col 5 to line %d, col %d of module VSR" % (i + 2, i + 3, len(lines[i + 2]))
