"""CPU: the OSPFv2, OSPFv3 and IS-IS route tables share one library.  Building them in any order gives the same
tables, and the route stage's C signatures do not depend on which class was built last."""
from holo_b200 import capi, isis, ospfv2, ospfv3, synth
from isis_synth import synth_instance


def test_tables_and_signatures_do_not_depend_on_build_order(built):
    t = synth.random_topology(60, 240, synth.SEED_BASE + 71, cost_choices=[5, 10], lan_fraction=0.1)
    build = {
        "ospfv2": lambda: ospfv2.RouteTable(ospfv2.Flat(ospfv2.synth_area(t, root=0, sr=True))),
        "ospfv3": lambda: ospfv3.RouteTable(ospfv3.Flat(ospfv3.synth_area(t, root=0))),
        "isis": lambda: isis.RouteTable(synth_instance(t, 0, sr=True)),
    }
    lib = capi.load_library()
    tables, argtypes = {}, []
    for order in (("ospfv3", "ospfv2", "isis"), ("isis", "ospfv2", "ospfv3"), ("ospfv2", "ospfv3", "isis")):
        for kind in order:
            rt = build[kind]()
            arrays = [rt.prefix.tobytes(), (rt.len if kind == "isis" else rt.plen).tobytes(), rt.off.tobytes(),
                      rt.contribs.tobytes(), rt.n_prefixes, rt.n_contributors]
            assert rt.n_prefixes > 0 and rt.n_contributors >= rt.n_prefixes
            assert tables.setdefault(kind, arrays) == arrays, kind
            argtypes.append(lib.hspf_ospfv2_rtable_arrays.argtypes)
    assert all(a == argtypes[0] for a in argtypes)
