"""Host-side mirror of the reference's ``gnn/models``: ``ReaRev`` and ``NSM`` with the reference's
constructor ``Model(args, num_entity, num_relation, num_word)``, ``forward(batch, training=False) ->
(loss, pred, pred_dist, tp_list)``, parameter names (checkpoint layout ``{'model_state_dict': ...}``,
gnn/train_model.py:236-252) and config keys (gnn/parsing.py) -- so the module drops into
``Trainer_KBQA`` / ``Evaluator`` (gnn/train_model.py:49-57, gnn/evaluate.py:160).

  BaseModel   gnn/models/base_model.py:10-297
  ReaRev      gnn/models/ReaRev/rearev.py:19-244
  NSM         gnn/models/NSM/nsm.py:19-254
  GraftNet    gnn/models/GraftNet/graftnet.py:21-183

``model(batch)`` runs the hand-written CUDA path; ``model(batch, training=True)`` -- what ``Trainer_KBQA.train_epoch``
calls (gnn/train_model.py:222) -- evaluates the same math with differentiable torch ops on the same parameters
(autograd_path.py) and returns ``tp_list = [h1, f1]`` like the reference (rearev.py:238-241), so the import swap of
INTEGRATION.md leaves training working.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import autograd_path, batching, ops
from .modules import (AttnEncoder, BERTInstruction, Fusion, GraftLayer, LSTMInstruction, NSMLayer, QueryReform,
                      ReasonGNNLayer, TypeLayer)

VERY_SMALL_NUMBER = 1e-10


def _no_autocast():
    """Inference runs the project's fp32 kernels whatever torch.autocast says around it: an enabled autocast would
    otherwise hand bf16 / fp16 activations from the torch-side GEMMs to kernels that take fp32, and the results must
    not depend on it."""
    return torch.autocast("cuda", enabled=False)


class BaseModel(nn.Module):
    def __init__(self, args, num_entity, num_relation, num_word):
        super().__init__()
        self.num_relation, self.num_entity, self.num_word = num_relation, num_entity, num_word
        self.kge_frozen = args["kge_frozen"]
        self.kg_dim = args["kg_dim"]
        self.entity_emb_file = args["entity_emb_file"]
        self.relation_emb_file = args["relation_emb_file"]
        self.relation_word_emb = args["relation_word_emb"]
        self.word_emb_file = args["word_emb_file"]
        self.entity_dim = args["entity_dim"]
        self.lm = args["lm"]
        if self.lm in ["bert"]:
            args["word_dim"] = 768
        self.word_dim = args["word_dim"]
        self.rel_texts = None
        self.device = torch.device("cuda" if args["use_cuda"] else "cpu")
        for k, v in args.items():                                  # base_model.py:50-57
            if k.endswith("dim"):
                setattr(self, k, v)
            if k.endswith("emb_file") or k.endswith("kge_file"):
                setattr(self, k, None if v is None else args["data_folder"] + v)
        self.use_inverse_relation = args.get("use_inverse_relation", False)
        self.use_self_loop = args.get("use_self_loop", True)
        self.eps = args["eps"]
        self.loss_type = args.get("loss_type", "kl")
        self.norm_rel = args["norm_rel"]
        self.normalized_gnn = args["normalized_gnn"]
        self._embedding_def()
        args["word_dim"] = self.word_dim

    # base_model.py:70-146
    def _embedding_def(self):
        ne, nr, nw = self.num_entity, self.num_relation, self.num_word
        if self.lm != "lstm":
            self.word_dim = 768
            self.word_embedding = nn.Embedding(nw + 1, self.word_dim, padding_idx=nw)
        elif self.word_emb_file is not None:
            word_emb = np.load(self.word_emb_file)
            self.word_dim = word_emb.shape[1]
            self.word_embedding = nn.Embedding(nw + 1, self.word_dim, padding_idx=nw)
            self.word_embedding.weight = nn.Parameter(
                torch.from_numpy(np.pad(word_emb, ((0, 1), (0, 0)), "constant")).float(),
                requires_grad=False)
        else:
            self.word_embedding = nn.Embedding(nw + 1, self.word_dim, padding_idx=nw)
        if self.entity_emb_file is not None:
            self.encode_type = False
            emb = np.load(self.entity_emb_file)
            ent_num, self.ent_dim = emb.shape
            self.entity_embedding = nn.Embedding(ne + 1, self.ent_dim, padding_idx=ne)
            if ent_num == ne:
                self.entity_embedding.weight = nn.Parameter(
                    torch.from_numpy(np.pad(emb, ((0, 1), (0, 0)), "constant")).float())
            self.entity_embedding.weight.requires_grad = not self.kge_frozen
        else:
            self.ent_dim = self.kg_dim
            self.encode_type = True
        if self.relation_emb_file is not None:
            half = np.load(self.relation_emb_file)
            full = np.concatenate([half, half]) if self.use_inverse_relation else half
            np_tensor = np.pad(full, ((0, 2 if self.use_self_loop else 0), (0, 0)), "constant")
            rel_num, self.rel_dim = np_tensor.shape
            self.relation_embedding = nn.Embedding(nr + 1, self.rel_dim)
            if rel_num == nr:
                self.relation_embedding.weight = nn.Parameter(torch.from_numpy(np_tensor).float())
            self.relation_embedding.weight.requires_grad = not self.kge_frozen
        elif self.relation_word_emb:
            self.rel_dim = self.entity_dim
            self.relation_embedding = nn.Embedding(nr + 1, self.rel_dim)
            self.relation_embedding_inv = nn.Embedding(nr + 1, self.rel_dim)
        else:
            self.rel_dim = 2 * self.kg_dim
            self.relation_embedding = nn.Embedding(nr + 1, self.rel_dim)
            self.relation_embedding_inv = nn.Embedding(nr + 1, self.rel_dim)

    def encode_rel_texts(self, rel_texts, rel_texts_inv):          # base_model.py:168-176
        self.rel_texts = torch.from_numpy(rel_texts).long().to(self.device)
        self.rel_texts_inv = torch.from_numpy(rel_texts_inv).long().to(self.device)
        self.instruction.eval()
        with torch.no_grad():
            self.rel_features = self.instruction.encode_question(self.rel_texts, store=False)
            self.rel_features_inv = self.instruction.encode_question(self.rel_texts_inv, store=False)

    def _make_instruction(self, args):                             # rearev.py:121-127 / nsm.py:70-76
        if args["lm"] == "lstm":
            return LSTMInstruction(args, self.word_embedding, self.num_word)
        return BERTInstruction(args, self.word_embedding, self.num_word, args["lm"])

    def _rel_text_features(self, raw, texts, att):
        """Relation-text branch of get_rel_feature (rearev.py:100-111 / nsm.py:104-111): project the stored encoder
        states of the relation names and pool them with ``att`` over the non-pad tokens."""
        ins = self.instruction
        if not hasattr(ins, "question_emb"):
            raise NotImplementedError(
                "relation_word_emb needs a language-model encoder (--lm sbert/bert/...): with --lm lstm the reference "
                "itself fails here (LSTMInstruction has no question_emb, rearev.py:101)")
        return att(ins.question_emb(raw), (texts != ins.pad_val).float())

    def _get_ent_init(self, db, rel_features, layer):              # rearev.py:79-88 / nsm.py:84-94
        """Initial node embeddings, written straight into the reasoning layer's h slot(s)."""
        planes = layer.cur_planes()
        if planes is not None:
            planes = tuple(p[:, : self.entity_dim] for p in planes)
            out = layer.h32
        else:
            out = layer.h_view
        if self.encode_type:
            # in planes mode nothing reads the fp32 h before the first e2e GEMM rewrites it
            self.type_layer(db.graph, rel_features, None if planes is not None else out, planes)
            if planes is not None:
                layer.h32_valid = False
        else:
            emb = self.entity_embedding(db.local_entity).view(db.B * db.N, -1).contiguous()
            ops.linear(emb, self.entity_linear.weight, self.entity_linear.bias, out=out)
            if planes is not None:
                ops.split_bf16(out, planes[0], planes[1])
                layer.h32_valid = True
        return out

    # base_model.py:186-215 + rearev.py:156-160
    def calc_loss_label(self, curr_dist, teacher_dist, label_valid):
        if self.loss_type == "bce":
            tgt = (teacher_dist > 0).float() * 0.9
            tp = F.binary_cross_entropy_with_logits(curr_dist, tgt, reduction="none")
        else:
            answer_len = torch.sum(teacher_dist, dim=1, keepdim=True)
            answer_len = torch.where(answer_len == 0, torch.ones_like(answer_len), answer_len)
            tp = F.kl_div(torch.log(curr_dist + 1e-8), teacher_dist / answer_len, reduction="none")
        return torch.sum(tp * label_valid) / curr_dist.size(0)

    def _loss_and_pred(self, pred_dist, answer_dist):             # rearev.py:228-232 / nsm.py:236-243
        if self.loss_type == "kl":
            return ops.kl_loss_pred(pred_dist, answer_dist)
        case_valid = (torch.sum(answer_dist, dim=1, keepdim=True) > 0).float()
        return self.calc_loss_label(pred_dist, answer_dist, case_valid), torch.max(pred_dist, dim=1)[1]

    FORK_QUESTION_SIDE = True

    def _fork_instructions(self, q_input):
        """Run the instruction encoder on a side stream; pair with :meth:`_join_instructions`."""
        if not self.FORK_QUESTION_SIDE:
            return self.instruction(q_input)
        cur = torch.cuda.current_stream()
        side = getattr(self, "_side_stream", None)
        if side is None or side.device != cur.device:
            side = self._side_stream = torch.cuda.Stream(device=cur.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            ins = self.instruction(q_input)
        return ins

    def _join_instructions(self, ins):
        if self.FORK_QUESTION_SIDE:
            cur = torch.cuda.current_stream()
            cur.wait_stream(self._side_stream)
            # tensors produced on the side stream and read on this one from now on
            enc = self.instruction
            for t in (ins, getattr(enc, "query_hidden_emb", None), getattr(enc, "query_node_emb", None),
                      getattr(enc, "relational_ins", None)):
                if isinstance(t, torch.Tensor) and t.is_cuda:
                    t.record_stream(cur)
        return ins

    def _check_ready(self):
        dev = self.word_embedding.weight.device
        if dev.type != "cuda":
            raise RuntimeError("gnn_rag_b200 models run on a CUDA device only (no CPU fallback); "
                               "construct with args['use_cuda']=True / call .cuda()")
        return dev


class ReaRev(BaseModel):
    def __init__(self, args, num_entity, num_relation, num_word):
        super().__init__(args, num_entity, num_relation, num_word)
        D = self.entity_dim
        self.num_iter, self.num_ins, self.num_gnn = args["num_iter"], args["num_ins"], args["num_gnn"]
        self.alg = args["alg"]
        assert self.alg == "bfs"
        self.linear_dropout = args["linear_dropout"]
        self.entity_linear = nn.Linear(self.ent_dim, D)
        self.relation_linear = nn.Linear(self.rel_dim, D)
        self.linear_drop = nn.Dropout(p=self.linear_dropout)
        if self.encode_type:
            self.type_layer = TypeLayer(D, D, self.linear_drop, self.device, self.norm_rel)
        self.self_att_r = AttnEncoder(D)
        self.reasoning = ReasonGNNLayer(args, num_entity, num_relation, D, self.alg)
        self.instruction = self._make_instruction(args)
        if args["lm"] == "lstm":
            self.relation_linear = nn.Linear(D, D)               # rearev.py:125
        self.lin = nn.Linear(3 * D, D)                           # unused in forward (checkpoint compat)
        self.fusion = Fusion(D)                                  # unused in forward (checkpoint compat)
        for i in range(self.num_ins):
            self.add_module("reform" + str(i), QueryReform(D))
        self.to(self.device)

    def get_rel_feature(self):                                   # rearev.py:91-111
        """-> ops.RelFeatures with the forward and inverse relation features stacked [2*R1, D]."""
        if self.rel_texts is None:
            lin = self.relation_linear
            return ops.rel_features_from_embeddings(
                [self.relation_embedding.weight, self.relation_embedding_inv.weight], lin.weight, lin.bias)
        rel, rel_inv = self.get_rel_feature_train()
        return ops.rel_features_from_tensors([rel.contiguous(), rel_inv.contiguous()])

    def get_rel_feature_train(self):
        """(rel_features, rel_features_inv) as plain fp32 tensors with autograd (rearev.py:91-111)."""
        if self.rel_texts is None:
            lin = self.relation_linear
            return lin(self.relation_embedding.weight), lin(self.relation_embedding_inv.weight)
        # both directions are masked with rel_texts, as in the reference (:104-105)
        return (self._rel_text_features(self.rel_features, self.rel_texts, self.self_att_r),
                self._rel_text_features(self.rel_features_inv, self.rel_texts, self.self_att_r))

    def forward(self, batch, training=False):
        """rearev.py:163-243.  ``batch`` = the ``get_batch`` tuple (host numpy) or a pre-staged
        :class:`batching.DeviceBatch`.  ``training=True``: differentiable torch path (autograd_path.py)."""
        if training:
            return autograd_path.rearev_forward(self, batch)
        with torch.no_grad(), _no_autocast():
            return self._forward_infer(batch)

    def _forward_infer(self, batch):
        dev = self._check_ready()
        D, I = self.entity_dim, self.num_ins
        db = batching.stage_batch(batch, dev, self.num_relation + 1, self.normalized_gnn, self.norm_rel)
        self.last_batch = db
        B, N = db.B, db.N
        # the question side (embedding -> LSTM / LM -> instruction attention) does not depend on the graph side (relation
        # features, hoisted tables, TypeLayer): fork it onto a second stream (captured as a parallel branch by GraphedStep)
        instructions = self._fork_instructions(db.q_input)
        rel_f = self.get_rel_feature()                           # both directions, stacked
        self.reasoning.init_reason(db, rel_f)
        self._get_ent_init(db, rel_f, self.reasoning)           # TypeLayer straight into the h slot
        instructions = self._join_instructions(instructions)     # rearev.py:192-196
        self.dist_history = [db.seed_dist]
        h = None
        reforms = [getattr(self, "reform" + str(j)).fusion for j in range(I)]
        Wr, Wg = [f.r.weight for f in reforms], [f.g.weight for f in reforms]
        seed_rows = db.query_entities.reshape(-1)                # the rows of h the reform reads
        for t in range(self.num_iter):                           # rearev.py:206-221
            last_iter = t == self.num_iter - 1
            relation_ins = instructions                          # [B, I, D]
            dist = db.seed_dist                                  # distribution resets to the seed (:208)
            for j in range(self.num_gnn):                        # only the last layer's h feeds the reform
                last = j == self.num_gnn - 1
                # j == 0: the prior is the seed distribution (non-zero on a few nodes) -> sparse-prior path.  The last
                # layer of the last iteration leaves the full fp32 h (layer.h_view) and no planes for a next layer;
                # the one of an earlier iteration writes fp32 h on the seed rows only
                dist, hj = self.reasoning(dist, relation_ins, step=j, need_h=last, sparse_prior=(j == 0),
                                          h_rows=seed_rows if last and not last_iter else None,
                                          next_layer=not (last and last_iter))
                h = hj if hj is not None else h
            self.dist_history.append(dist)
            if not last_iter:                                    # the last reform's instructions are never read
                # all num_ins reforms (seed_retrieve + Fusion) in one launch
                instructions = ops.query_reform(db.query_entities, h, instructions, Wr, Wg, B, N)
        pred_dist = self.dist_history[-1]
        loss, pred = self._loss_and_pred(pred_dist, db.answer_dist)
        return loss, pred, pred_dist, None


class NSM(BaseModel):
    def __init__(self, args, num_entity, num_relation, num_word):
        super().__init__(args, num_entity, num_relation, num_word)
        D = self.entity_dim
        self.num_step = args["num_step"]
        self.num_iter = self.num_step
        self.model_name = args["model_name"].lower()
        self.lambda_constrain, self.lambda_back = args["lambda_constrain"], args["lambda_back"]
        if self.lambda_back != 0.0 or self.lambda_constrain != 0.0:
            raise NotImplementedError("NSM backward-consistency branch is broken in the reference "
                                      "(nsm_gnn.py:122 reads an unset attribute); not reproduced")
        self.linear_dropout = args["linear_dropout"]
        self.entity_linear = nn.Linear(self.ent_dim, D)
        self.relation_linear1 = nn.Linear(self.rel_dim, D)
        self.relation_linear2 = nn.Linear(self.rel_dim, D)       # unused in forward
        self.kg_lin = nn.Linear(D, D)                            # unused in forward
        self.score_func = nn.Linear(2 * D, 1)                    # unused in forward
        self.linear_drop = nn.Dropout(p=self.linear_dropout)
        if self.encode_type:
            self.type_layer = TypeLayer(D, D, self.linear_drop, self.device, self.norm_rel)
        self.self_att_r = AttnEncoder(D)
        self.self_att_r2 = AttnEncoder(D)
        self.reasoning = NSMLayer(args, num_entity, num_relation, D)
        self.reasoning2 = NSMLayer(args, num_entity, num_relation, D)   # unused in forward (ckpt compat)
        self.instruction = self._make_instruction(args)
        self.to(self.device)

    def get_rel_feature(self):                                   # nsm.py:97-111
        if self.rel_texts is None:
            lin = self.relation_linear1
            return ops.rel_features_from_embeddings([self.relation_embedding.weight], lin.weight, lin.bias)
        return ops.rel_features_from_tensors([self.get_rel_feature_train().contiguous()])

    def get_rel_feature_train(self):
        if self.rel_texts is None:
            return self.relation_linear1(self.relation_embedding.weight)
        return self._rel_text_features(self.rel_features, self.rel_texts, self.self_att_r)

    def forward(self, batch, training=False):
        """nsm.py:179-254 (forward reasoning only).  ``training=True``: differentiable torch path."""
        if training:
            return autograd_path.nsm_forward(self, batch)
        with torch.no_grad(), _no_autocast():
            return self._forward_infer(batch)

    def _forward_infer(self, batch):
        dev = self._check_ready()
        db = batching.stage_batch(batch, dev, self.num_relation + 1, self.normalized_gnn, self.norm_rel)
        self.last_batch = db
        instruction_list = self._fork_instructions(db.q_input)
        rel_f = self.get_rel_feature()
        self.reasoning.init_reason(db, rel_f)
        self._get_ent_init(db, rel_f, self.reasoning)
        instruction_list = self._join_instructions(instruction_list)
        dist = db.seed_dist
        self.dist_history = [dist]
        for i in range(self.num_step):                           # nsm.py:219-222
            dist = self.reasoning(dist, instruction_list[:, i], step=i)
            self.dist_history.append(dist)
        pred_dist = self.dist_history[-1]
        loss, pred = self._loss_and_pred(pred_dist, db.answer_dist)
        return loss, pred, pred_dist, None


class GraftNet(BaseModel):
    """GraftNet (graftnet.py:21-183) on the 9-tuple of GraftSingleDataLoader.get_batch (10 with ``test=True``,
    dataset_load_graft.py:113-149).  ``model(batch)`` runs the CUDA path (csrc/graft.cu + the wgmma GEMMs);
    ``model(batch, training=True)`` the differentiable restatement of autograd_path.graftnet_forward."""

    def __init__(self, args, num_entity, num_relation, num_word):
        super().__init__(args, num_entity, num_relation, num_word)
        D = self.entity_dim
        self.num_layer = args["num_layer"]
        self.loss_type = args["loss_type"]
        self.model_name = args["model_name"].lower()
        self.lm = args["lm"]
        self.norm_rel = args["norm_rel"]
        self.num_iter = self.num_layer
        self.linear_dropout = args["linear_dropout"]
        self.entity_linear = nn.Linear(self.ent_dim, D)
        self.relation_linear1 = nn.Linear(self.rel_dim, D)
        self.linear_drop = nn.Dropout(p=self.linear_dropout)
        if self.encode_type:
            self.type_layer = TypeLayer(D, D, self.linear_drop, self.device, self.norm_rel)
        self.self_att_r = AttnEncoder(D)
        self.reasoning = GraftLayer(args, num_entity, num_relation, D)
        self.instruction = self._make_instruction(args)
        if args["lm"] != "lstm":
            self.relation_linear = nn.Linear(self.word_dim, D)    # graftnet.py:72 (unused in forward)
        self.to(self.device)

    def get_rel_feature_train(self):                               # graftnet.py:85-102
        if self.rel_texts is None:
            return self.relation_linear1(self.relation_embedding.weight)
        if self.lm == "lstm":
            raise NotImplementedError("relation texts with --lm lstm: the reference pools the relation states twice "
                                      "and fails (graftnet.py:96-98)")
        return self._rel_text_features(self.rel_features, self.rel_texts, self.self_att_r)

    def get_rel_feature(self):
        """fp32 relation features [R1, D]."""
        if self.rel_texts is None:
            lin = self.relation_linear1
            return ops.rel_linear(self.relation_embedding.weight, lin.weight, lin.bias)
        return self.get_rel_feature_train().contiguous()

    def forward(self, batch, training=False):
        """graftnet.py:135-183 -> (loss, pred, pred_dist, tp_list)."""
        if training:
            return autograd_path.graftnet_forward(self, batch)
        with torch.no_grad(), _no_autocast():
            return self._forward_infer(batch)

    def _init_h(self, db, rel):                                    # graftnet.py:74-83
        layer = self.reasoning
        planes = layer.h_planes()
        if self.encode_type:
            self.type_layer(db.graph, ops.rel_features_from_tensors([rel]), layer.h32, planes)
        else:
            emb = self.entity_embedding(db.local_entity).view(db.B * db.N, -1).contiguous()
            ops.linear(emb, self.entity_linear.weight, self.entity_linear.bias, out=layer.h32)
            ops.split_bf16(layer.h32, planes[0], planes[1])

    def _forward_infer(self, batch, check_status=True):
        """``check_status=False``: skip the read-back of the staging status words (a host sync) -- for a caller that
        reads ``db.graft.status`` / ``db.graph.status`` itself after the step (GraphedStep captures this forward)."""
        dev = self._check_ready()
        db = batching.stage_graft_batch(batch, dev, self.num_relation + 1, self.normalized_gnn, self.norm_rel)
        self.last_batch = db
        enc = self.instruction
        enc.encode_question(db.q_input)                            # graftnet.py:108-111 (the instructions are unused)
        qh = enc.query_hidden_emb.contiguous()
        qnode = enc.query_node_emb.reshape(db.B, -1)
        rel = self.get_rel_feature()
        layer = self.reasoning
        layer.init_reason(db, rel, qh, enc.query_mask)
        self._init_h(db, rel)
        dist = db.seed_dist
        self.dist_history = [dist]
        self.pagerank_history = [dist]
        query = qnode
        for i in range(self.num_layer):                            # graftnet.py:163-165
            score, dist, query = layer(dist, query, i, last=(i == self.num_layer - 1))
            self.dist_history.append(score)
            self.pagerank_history.append(dist)
        pred_dist = self.dist_history[-1]
        case_valid = (torch.sum(db.answer_dist, dim=1, keepdim=True) > 0).float()
        loss = self.calc_loss_label(layer.logits(), db.answer_dist, case_valid)
        pred = torch.max(pred_dist, dim=1)[1]
        if check_status:
            db.graft.check_status()
        return loss, pred, pred_dist, None
