"""Hand-built cases of preemption under the PodFitsHostPorts filter (include/bsched.h bs_upload_bound_host_ports),
each with its answers written out.  A case is (snapshot, bound-pod table, cols, bound_ports, preemptor pod indices,
walk, gang, expected): cols as host_ports_ref.random_columns gives them, bound_ports [V] uint64, and expected per
preemptor (node, victims, n_candidates) for bs_preempt or (node, victims, n_candidates, outcome) for the walk.  Lanes
as in tests/preempt_cases.py; every node is full on cpu (10 of 10) unless a case says otherwise, and preemptors ask
for no cpu, so ports decide."""
import numpy as np

import preempt_cases
import pdb_cases

NONE, NOMINATED, ROLLED_BACK = range(3)   # BS_WALK_*
TCP, UDP = 0, 1
ANY = 0   # BS_HOSTPORT_IP_ANY
# E0 0.0.0.0:8080/TCP, E1 ip1:8080/TCP, E2 ip2:8080/TCP, E3 0.0.0.0:8080/UDP, E4 0.0.0.0:22/TCP
ENTRIES = [(ANY, TCP, 8080), (1, TCP, 8080), (2, TCP, 8080), (ANY, UDP, 8080), (ANY, TCP, 22)]
E0, E1, E2, E3, E4 = (1 << k for k in range(5))


def _case(nodes, used, pods, want, rows, ports, pick, walk=False, gang=False, expected=()):
    snap = preempt_cases._snap(nodes, pods)
    bound = pdb_cases._bound(rows)
    cols = ((np.array(ENTRIES, np.int64), np.array(used, np.uint64)), np.array(want, np.uint64))
    return snap, bound, cols, np.array(ports, np.uint64), list(pick), walk, gang, list(expected)


def cases():
    c = {}
    full = {"cpu_alloc": 10, "cpu_req": 10}
    # Row 1 (prio 1, cpu 1) holds port 22; rows 0 and 2 hold more cpu and no port.  The pod needs no cpu: every row is
    # reprieved but the port holder.
    c["victim_only_for_its_port"] = _case(
        [full], [E4], [{"prio": 100}], [E4],
        [{"node": 0, "cpu": 5, "prio": 5}, {"node": 0, "cpu": 1, "prio": 1}, {"node": 0, "cpu": 4, "prio": 3}],
        [0, E4, 0], [0], expected=[(0, [1], 1)])
    # Node 0's port is held by a prio-200 row, which no prio-100 preemptor may evict: the node drops out, and the
    # candidates shrink to node 1.  Without the filter node 0 would win at once (no victims).
    c["higher_priority_holder_drops_node"] = _case(
        [full, full], [E4, E4], [{"prio": 100}], [E4],
        [{"node": 0, "prio": 200}, {"node": 1, "prio": 1}], [E4, E4], [0], expected=[(1, [1], 1)])
    # The wildcard rule against a node using ip1:8080/TCP (row 0): ip2:8080/TCP and 0.0.0.0:8080/UDP pass,
    # 0.0.0.0:8080/TCP conflicts.
    c["wildcard_specific_ip_and_protocol"] = _case(
        [full], [E1], [{"prio": 100}] * 3, [E2, E0, E3],
        [{"node": 0, "prio": 1}], [E1], [0, 1, 2], expected=[(0, [], 1), (0, [0], 1), (0, [], 1)])
    # A node using the wildcard 0.0.0.0:8080/TCP (row 0) conflicts with ip1:8080/TCP.
    c["wildcard_on_the_node"] = _case(
        [full], [E0], [{"prio": 100}], [E1], [{"node": 0, "prio": 1}], [E0], [0], expected=[(0, [0], 1)])
    # Rows 0 (prio 200) and 1 (prio 1) both list port 22.  Removing row 1 deletes the entry from the set although row
    # 0 still holds it (HostPortInfo.Remove): the node is a candidate and row 1 is the only victim.
    c["set_delete_quirk"] = _case(
        [full], [E4], [{"prio": 100}], [E4],
        [{"node": 0, "prio": 200}, {"node": 0, "prio": 1}], [E4, E4], [0], expected=[(0, [1], 1)])
    # Node 0 uses port 22 but no bound row holds it (say a pod outside the table): nothing frees it, node 1 wins.
    c["used_entry_no_row_holds"] = _case(
        [full, full], [E4, E4], [{"prio": 100}], [E4],
        [{"node": 0, "prio": 1}, {"node": 1, "prio": 1}], [0, E4], [0], expected=[(1, [1], 1)])
    # Budgets and ports.  The pod asks for cpu 5 and port 22.  Node 0: the violating row 0 is reprieved, row 1 (port
    # 22) goes.  Node 1: the violating row 2 holds the port and goes; row 3 is reprieved.  Node 0 has fewer violating
    # victims and wins.
    c["ports_and_pdb_violating_rows"] = _case(
        [full, full], [E4, E4], [{"prio": 100, "cpu": 5}], [E4],
        [{"node": 0, "cpu": 5, "prio": 1, "vio": True}, {"node": 0, "cpu": 5, "prio": 2},
         {"node": 1, "cpu": 5, "prio": 1, "vio": True}, {"node": 1, "cpu": 5, "prio": 2}],
        [0, E4, E4, 0], [0], expected=[(0, [1], 2)])
    # The walk: p0 is nominated to node 0 without victims; its port keeps p1, who wants the same, off node 0.
    c["walk_nominated_port_blocks_second"] = _case(
        [full, full], [0, 0], [{"prio": 100}] * 2, [E4, E4],
        [{"node": 0, "prio": 1}, {"node": 1, "prio": 1}], [0, 0], [0, 1], walk=True,
        expected=[(0, [], 2, NOMINATED), (1, [], 1, NOMINATED)])
    # The walk: p0 evicts row 0, which holds the very port 22 p0 wants, and is nominated to node 0; p1 (cpu 5) then
    # evicts row 1 there.  Port 22 stays taken by the nominee, so p2, wanting it, finds no node: an engine that
    # nominated before it evicted would have deleted the nominee's own entry with row 0's.  (With priorities
    # non-increasing along the list, no row left on a nominee's node can hold an entry the nominee wants, since it
    # would have conflicted with it, so keeping the nominated mask apart from the bound one cannot change an answer
    # beyond this; the walk keeps them apart because that is upstream's model.)
    c["walk_eviction_keeps_nominated_port"] = _case(
        [full], [E4 | E1], [{"prio": 100}, {"prio": 100, "cpu": 5}, {"prio": 100}], [E4, 0, E4],
        [{"node": 0, "prio": 1}, {"node": 0, "prio": 1, "cpu": 10}], [E4, E1], [0, 1, 2], walk=True,
        expected=[(0, [0], 1, NOMINATED), (0, [1], 1, NOMINATED), (-1, [], 0, NONE)])
    # The walk with gang units: group 0's p0 evicts row 0 (prio 50, port 22) and keeps row 1 (prio 10, port
    # ip1:8080), which compaction moves into row 0's slot; p1 of the same group is kept off node 0 by p0's nominated
    # port, so the unit rolls back.  The online p2 then sees row 0 back with its port: it evicts row 0 alone.  A
    # rollback that left row 1's mask in row 0's slot would see no freeable port 22 there, and one that kept p0's
    # nominated port would see it taken: either gives p2 no node.
    c["walk_rolled_back_unit_gives_ports_back"] = _case(
        [full], [E4 | E1], [{"prio": 100, "gid": 0}, {"prio": 100, "gid": 0}, {"prio": 100}], [E4, E4, E4],
        [{"node": 0, "prio": 50, "gid": 1}, {"node": 0, "prio": 10, "gid": 1}], [E4, E1], [0, 1, 2], walk=True,
        gang=True, expected=[(-1, [], 1, ROLLED_BACK), (-1, [], 0, ROLLED_BACK), (0, [0], 1, NOMINATED)])
    # The same with p2 at priority 40, below row 0's 50: row 0 is no potential victim of p2, and its port 22, restored
    # to the node's used mask by the rollback, keeps p2 off node 0.  A rollback that did not restore the used mask
    # would leave it free and nominate p2 there without victims.  (Under gang units p2, a unit of one without a node,
    # reports ROLLED_BACK.)
    c["walk_rolled_back_unit_restores_used_ports"] = _case(
        [full], [E4], [{"prio": 100, "gid": 0}, {"prio": 100, "gid": 0}, {"prio": 40}], [E4, E4, E4],
        [{"node": 0, "prio": 50, "gid": 1}], [E4], [0, 1, 2], walk=True, gang=True,
        expected=[(-1, [], 1, ROLLED_BACK), (-1, [], 0, ROLLED_BACK), (-1, [], 0, ROLLED_BACK)])
    return c
