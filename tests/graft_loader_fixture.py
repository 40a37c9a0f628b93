"""Stand-in loader states for GraftNet's batch assembly (gnn/dataset_load_graft.py:27-102 on top of
gnn/dataset_load.py:473-527): per-question subgraph tuples in the three forms ``create_kb_adj_mats_facts`` parses
(entity / relation names, ``{'text': ...}`` dicts, integer local ids), the name -> id maps, the global -> local entity
maps, ``max_facts`` and the fields ``_build_fact_mat`` reads.

``GraftStandIn`` holds the state only.  tests/golden/make_graft_fact_mat_golden.py binds the unmodified reference
methods to it; the host tests replay the reference's per-question ``create_kb_adj_mats_facts`` results recorded in the
golden files (:class:`ReplayGraftLoader`), so they run without the reference checkout."""
import numpy as np

from loader_fixture import FakeLoader


class GraftStandIn(FakeLoader):
    def __init__(self, seed, num_questions, max_local_entity, num_relations, form, use_inverse_relation=False,
                 facts_hi=30, empty=()):
        rs = np.random.RandomState(seed)
        num_kb_relation = (2 if use_inverse_relation else 1) * num_relations + 1     # dataset_load.py:119-124
        super().__init__(seed, num_questions, max_local_entity, num_kb_relation, facts_hi=facts_hi)
        self.use_inverse_relation = use_inverse_relation
        self.relation2id = {"rel.%d" % k: k for k in range(num_relations)}
        self.entity2id = {}
        self.data = []
        self.global2local_entity_maps = []
        max_tuples = 0
        for q in range(num_questions):
            n_ent = int(rs.randint(2, max_local_entity + 1))
            ents = rs.choice(10 * max_local_entity, n_ent, replace=False)
            g2l = {}
            for k, e in enumerate(ents.tolist()):
                self.entity2id.setdefault("ent.%d" % e, e)
                g2l[e] = k
            self.global2local_entity_maps.append(g2l)
            T = 0 if q in empty else int(rs.randint(1, facts_hi + 1))
            max_tuples = max(max_tuples, T)
            tuples = []
            for _ in range(T):
                h, t = (int(x) for x in rs.choice(ents, 2))
                r = int(rs.randint(0, num_relations))
                if form == "str":
                    tuples.append(["ent.%d" % h, "rel.%d" % r, "ent.%d" % t])
                elif form == "dict":
                    tuples.append([{"text": "ent.%d" % h}, {"text": "rel.%d" % r}, {"text": "ent.%d" % t}])
                elif form == "int":          # the bare-except fallback: ids already global, relation as an int string
                    tuples.append([h, str(r), t])
                else:
                    raise ValueError(form)
            self.data.append({"subgraph": {"tuples": tuples}})
        self.max_facts = 2 * max_tuples + max_local_entity                          # dataset_load.py:54, :72


CASES = {   # name -> (stand-in kwargs, sample_ids, fact_dropout, numpy seed)
    "str": (dict(seed=21, num_questions=6, max_local_entity=14, num_relations=7, form="str"), [0, 1, 2, 3, 4, 5],
            0.0, 31),
    "dict_dropout": (dict(seed=22, num_questions=7, max_local_entity=18, num_relations=5, form="dict"),
                     [6, 2, 2, 0, 5], 0.3, 32),
    "int_inverse": (dict(seed=23, num_questions=5, max_local_entity=12, num_relations=6, form="int",
                         use_inverse_relation=True), [4, 3, 1, 0], 0.0, 33),
    "str_inverse_dropout_empty": (dict(seed=24, num_questions=6, max_local_entity=10, num_relations=4, form="str",
                                       use_inverse_relation=True, empty=(2,)), [2, 0, 1, 5, 3], 0.3, 34),
    "dict_empty": (dict(seed=25, num_questions=4, max_local_entity=9, num_relations=3, form="dict", empty=(1,)),
                   [1, 3, 0], 0.0, 35),
}

# one get_batch: _build_fact_mat then _build_fact_mat_maxfacts on the same sample ids, under one seed
SEQUENCE = "dict_dropout"

PER_Q_KEYS = ("e2f_f", "e2f_e", "e2f_v", "f2e_e", "f2e_f", "f2e_v", "kb_fact_rel")
OUT_KEYS = ("mats0_batch", "mats0_0", "mats0_1", "vals0", "mats1_batch", "mats1_0", "mats1_1", "vals1",
            "kb_fact_rels")


def flatten_output(out):
    ((a, b, c, d), (e, f, g, h)), rels = out
    return dict(zip(OUT_KEYS, (a, b, c, d, e, f, g, h, rels)))


class ReplayGraftLoader(GraftStandIn):
    """The stand-in whose ``create_kb_adj_mats_facts`` returns the reference's recorded result for each sample (and
    counts its calls)."""

    def __init__(self, gold, **kw):
        super().__init__(**kw)
        self._gold = gold
        self.calls = 0

    def create_kb_adj_mats_facts(self, sample_id):
        self.calls += 1
        g = {k: self._gold["q%d_%s" % (sample_id, k)] for k in PER_Q_KEYS}
        return ((g["e2f_f"], g["e2f_e"], g["e2f_v"]), (g["f2e_e"], g["f2e_f"], g["f2e_v"])), g["kb_fact_rel"]
