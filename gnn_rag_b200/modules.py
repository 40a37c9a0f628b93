"""Host-side mirror of the reference's ``gnn/modules`` for the retrieval hot path.

Same class names, constructor arguments and parameter names as the reference so a reference
``state_dict`` loads unchanged (SURVEY.md 8b), but the graph work runs in the hand-written sm_90a kernels
behind the C ABI (ops.py) instead of ``index_select`` / ``Linear``-over-facts / ``torch.sparse.mm``:

  TypeLayer          gnn/modules/layer_init.py:8-65
  AttnEncoder/Fusion/QueryReform   gnn/modules/query_update.py:6-61
  LSTMInstruction    gnn/modules/question_encoding/{base,lstm}_encoder.py  (stays in PyTorch: O(B*Q*D), it
                     feeds the path, SURVEY.md 8a row 12)
  ReasonGNNLayer     gnn/modules/kg_reasoning/reasongnn.py:11-174
  NSMLayer           gnn/modules/kg_reasoning/nsm_gnn.py:14-112
  GraftLayer         gnn/modules/kg_reasoning/graft_gnn.py:14-153
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops

VERY_NEG_NUMBER = -100000000000


class TypeLayer(nn.Module):
    """h0[n] = relu(sum_{f: tail=n} v_f W rel[r_f] + sum_{f: head=n} v_f W rel[r_f])  (layer_init.py:25-62).
    ``kb_self_linear`` is applied to the R1 relation rows once (hoisted) instead of to F gathered rows."""

    def __init__(self, in_features, out_features, linear_drop, device, norm_rel):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.linear_drop = linear_drop
        self.kb_self_linear = nn.Linear(in_features, out_features)
        self.device = device
        self.norm_rel = norm_rel

    def forward(self, graph, rel_features, out, planes=None):
        """``rel_features``: ops.RelFeatures (only the forward direction is used, layer_init.py:39-41)."""
        table = ops.rel_table(rel_features, self.kb_self_linear.weight, self.kb_self_linear.bias, dirs=1)[0]
        wt, wh = (graph.wr_t, graph.wr_h) if self.norm_rel else (None, None)
        ops.type_layer(graph, table, out, wt, wh, planes=planes)
        return out


class AttnEncoder(nn.Module):
    """query_update.py:46-61 (relation-text pooling; dense, stays in PyTorch)."""

    def __init__(self, d_hid):
        super().__init__()
        self.attn_linear = nn.Linear(d_hid, 1, bias=False)

    def forward(self, x, x_mask):
        a = self.attn_linear(x) - (1 - x_mask.unsqueeze(2)) * 1e8
        return (x * F.softmax(a, dim=1)).sum(1)


class Fusion(nn.Module):
    """query_update.py:6-16: gate between instruction x and retrieved seed embedding y."""

    def __init__(self, d_hid):
        super().__init__()
        self.r = nn.Linear(d_hid * 3, d_hid, bias=False)
        self.g = nn.Linear(d_hid * 3, d_hid, bias=False)

    def forward(self, x, y):
        z = torch.cat([x, y, x - y], dim=-1)
        g_ = torch.sigmoid(self.g(z))
        return g_ * self.r(z) + (1 - g_) * x


class QueryReform(nn.Module):
    """query_update.py:18-44.  Only ``seed_retrieve`` reaches the output (the attention at :36-38 is dead
    code); the seed-weighted row pick runs in csrc/score.cu and touches only the seed rows."""

    def __init__(self, h_dim):
        super().__init__()
        self.fusion = Fusion(h_dim)
        self.q_ent_attn = nn.Linear(h_dim, h_dim)   # kept for state_dict compatibility

    def forward(self, q_node, h_view, seed_info, B, N):
        seed_retrieve = ops.seed_retrieve(seed_info, h_view, B, N, q_node.shape[1])
        return self.fusion(q_node, seed_retrieve)


class LSTMInstruction(nn.Module):
    """Question -> token states -> ``num_ins`` instruction vectors (lstm_encoder.py:10-45,
    base_encoder.py:73-114).  Dropouts are identity in eval mode (the only mode this path supports)."""

    def __init__(self, args, word_embedding, num_word):
        super().__init__()
        if "num_step" in args:                       # base_encoder.py:24-33
            self.num_ins = args["num_step"]
        elif "num_ins" in args:
            self.num_ins = args["num_ins"]
        elif "num_layer" in args:                  # GraftNet's CLI args carry only num_layer
            self.num_ins = args["num_layer"]
        else:
            self.num_ins = 1
        self.entity_dim = args["entity_dim"]
        self.word_dim = args["word_dim"]
        self.word_embedding = word_embedding
        self.num_word = num_word
        D = self.entity_dim
        self.node_encoder = nn.LSTM(input_size=self.word_dim, hidden_size=D, batch_first=True,
                                    bidirectional=False)
        self.cq_linear = nn.Linear(4 * D, D)
        self.ca_linear = nn.Linear(D, 1)
        for i in range(self.num_ins):
            self.add_module("question_linear" + str(i), nn.Linear(D, D))
        self.lstm_drop = nn.Dropout(p=args.get("lm_dropout", 0.0))        # base_encoder.py:49-52
        self.linear_drop = nn.Dropout(p=args.get("linear_dropout", 0.0))
        self.pad_val = num_word

    def encode_question_train(self, query_text):
        """lstm_encoder.py:32-45 with autograd (cuDNN / torch LSTM) -- the training path of autograd_path.py."""
        emb = self.lstm_drop(self.word_embedding(query_text))
        z = torch.zeros(1, query_text.size(0), self.entity_dim, device=emb.device, dtype=emb.dtype)
        hidden, (h_n, _c) = self.node_encoder(emb, (z, z.clone()))
        self.query_hidden_emb = hidden
        self.query_node_emb = h_n.squeeze(0).unsqueeze(1)
        self.query_mask_train = (query_text != self.num_word).float()

    def encode_question(self, query_text, store=True):
        emb = self.word_embedding(query_text)
        Bq = query_text.size(0)
        enc = self.node_encoder
        if emb.is_cuda and ops.lstm_ok(self.entity_dim):
            # input projection for all tokens at once (one GEMM), recurrence in one cluster kernel
            gx = F.linear(emb, enc.weight_ih_l0, enc.bias_ih_l0)
            hidden = ops.lstm_forward(gx, enc.weight_hh_l0, enc.bias_hh_l0)
            h_n = hidden[:, -1].unsqueeze(0)
        else:
            z = torch.zeros(1, Bq, self.entity_dim, device=emb.device, dtype=emb.dtype)
            with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):   # keep the encoder fp32-exact
                hidden, (h_n, c_n) = enc(emb, (z, z.clone()))
        if not store:
            return hidden
        self.query_node_emb = h_n.squeeze(0).unsqueeze(1)
        self.query_hidden_emb = hidden
        self._query_text = query_text
        return hidden, self.query_node_emb

    @property
    def query_mask(self):
        return (self._query_text != self.num_word).float()

    def init_reason(self, query_text):
        self.encode_question(query_text)
        self.relational_ins = torch.zeros(query_text.size(0), self.entity_dim, device=query_text.device)
        self.instructions = []

    def get_instruction(self, relational_ins, step=0):
        ri = relational_ins.unsqueeze(1)
        q_i = getattr(self, "question_linear" + str(step))(self.query_node_emb)
        cq = self.cq_linear(torch.cat((ri, q_i, q_i - ri, q_i * ri), dim=-1))
        ca = self.ca_linear(cq * self.query_hidden_emb)
        attn = F.softmax(ca + (1 - self.query_mask.unsqueeze(2)) * VERY_NEG_NUMBER, dim=1)
        return torch.sum(attn * self.query_hidden_emb, dim=1), attn

    def forward(self, query_text):
        """-> instructions [B, num_ins, D] (the reference returns the list of its num_ins slices)."""
        self.encode_question(query_text)
        I = self.num_ins
        lins = [getattr(self, "question_linear" + str(i)) for i in range(I)]
        ins = ops.instructions(self.query_hidden_emb, self.query_node_emb.squeeze(1), query_text, self.num_word,
                               [l.weight for l in lins], [l.bias for l in lins], self.cq_linear.weight,
                               self.cq_linear.bias, self.ca_linear.weight.view(-1), self.ca_linear.bias)
        self.relational_ins = ins[:, I - 1]
        return ins


# HuggingFace encoder variants of BERTInstruction (bert_encoder.py:29-60): name -> (hub id, config class, config
# overrides, word_dim, pad token id).  The architectures are fixed by the hub ids, so the encoder can be BUILT offline
# from its config; a published checkpoint then fills ``instruction.node_encoder.*`` through load_state_dict.
_LM_SPECS = {
    "bert": ("bert-base-uncased", "BertConfig", {}, 768, 0),
    "simcse": ("princeton-nlp/sup-simcse-bert-base-uncased", "BertConfig", {}, 768, 0),
    "relbert": ("pretrained_lms/sr-simbert/", "BertConfig", {}, 768, 0),
    "sbert": ("sentence-transformers/all-MiniLM-L6-v2", "BertConfig",
              dict(hidden_size=384, num_hidden_layers=6, num_attention_heads=12, intermediate_size=1536), 384, 0),
    "roberta": ("roberta-base", "RobertaConfig",
                dict(vocab_size=50265, max_position_embeddings=514, type_vocab_size=1, pad_token_id=1,
                     bos_token_id=0, eos_token_id=2, layer_norm_eps=1e-5), 768, 1),
    "sbert2": ("sentence-transformers/all-mpnet-base-v2", "MPNetConfig", dict(vocab_size=30527), 768, 1),
}


class BERTInstruction(nn.Module):
    """Language-model question encoder (bert_encoder.py:18-108) + the shared instruction attention
    (base_encoder.py:73-114).  Same parameter names as the reference (``node_encoder.*`` is the HuggingFace model,
    ``question_emb``, ``cq_linear``, ``ca_linear``, ``question_linear{i}``), so ``--lm sbert`` checkpoints load.

    The reference downloads tokenizer + weights from the hub at construction (:31-60,72).  Here the encoder is
    loaded from the local HuggingFace cache when it is there (``local_files_only``) and otherwise built from the
    architecture's config with random weights, to be filled by ``load_state_dict``; ``args['lm_config']`` (dict of
    config overrides, e.g. a 2-layer test model) takes precedence.  The transformer itself runs in PyTorch: it is
    the INPUT of the graph path (SURVEY 8a row 12); the instruction attention runs in csrc/question.cu."""

    def __init__(self, args, word_embedding, num_word, model):
        super().__init__()
        if model not in _LM_SPECS:
            raise NotImplementedError("lm=%r: supported language-model encoders are %s (t5 is an encoder-decoder "
                                      "the reference special-cases, bert_encoder.py:86-89)" % (model, sorted(_LM_SPECS)))
        if "num_step" in args:                       # base_encoder.py:24-33
            self.num_ins = args["num_step"]
        elif "num_ins" in args:
            self.num_ins = args["num_ins"]
        elif "num_layer" in args:                  # GraftNet's CLI args carry only num_layer
            self.num_ins = args["num_layer"]
        else:
            self.num_ins = 1
        self.model = model
        self.entity_dim = D = args["entity_dim"]
        self.word_embedding = word_embedding
        self.num_word = num_word
        self.lm_frozen = args.get("lm_frozen", 1)
        hub_id, cfg_cls, overrides, word_dim, pad = _LM_SPECS[model]
        self.pretrained_weights = hub_id
        self.word_dim = word_dim
        self.pad_val = pad
        self.cq_linear = nn.Linear(4 * D, D)
        self.ca_linear = nn.Linear(D, 1)
        for i in range(self.num_ins):
            self.add_module("question_linear" + str(i), nn.Linear(D, D))
        self.question_emb = nn.Linear(word_dim, D)
        self.lstm_drop = nn.Dropout(p=args.get("lm_dropout", 0.0))
        self.linear_drop = nn.Dropout(p=args.get("linear_dropout", 0.0))
        self.node_encoder = self._build_encoder(hub_id, cfg_cls, overrides, args.get("lm_config"))
        if self.node_encoder.config.hidden_size != word_dim:
            self.word_dim = self.node_encoder.config.hidden_size
            self.question_emb = nn.Linear(self.word_dim, D)
        for prm in self.node_encoder.parameters():                       # bert_encoder.py:74-81
            prm.requires_grad = self.lm_frozen != 1

    @staticmethod
    def _build_encoder(hub_id, cfg_cls, overrides, user_cfg):
        import transformers
        if user_cfg is None:
            try:
                return transformers.AutoModel.from_pretrained(hub_id, local_files_only=True)
            except Exception:  # noqa: BLE001 -- not in the local cache: build the architecture, weights come from the ckpt
                pass
        cfg = getattr(transformers, cfg_cls)(**dict(overrides, **(user_cfg or {})))
        return transformers.AutoModel.from_config(cfg)

    def _hidden(self, query_text):
        return self.node_encoder(query_text)[0]                          # bert_encoder.py:86 (no attention mask)

    def encode_question(self, query_text, store=True):                   # bert_encoder.py:83-105
        raw = self._hidden(query_text)
        if not store:
            return raw
        self.query_hidden_emb = self.question_emb(raw)
        self.query_node_emb = self.question_emb(raw[:, 0].unsqueeze(1))
        self._query_text = query_text
        return raw, self.query_node_emb

    def encode_question_train(self, query_text):
        self.encode_question(query_text)
        self.query_mask_train = (query_text != self.pad_val).float()

    @property
    def query_mask(self):
        return (self._query_text != self.pad_val).float()

    def forward(self, query_text):
        """-> instructions [B, num_ins, D]; the LM runs in torch, the attention steps in one kernel launch."""
        self.encode_question(query_text)
        I = self.num_ins
        lins = [getattr(self, "question_linear" + str(i)) for i in range(I)]
        ins = ops.instructions(self.query_hidden_emb.contiguous(), self.query_node_emb.squeeze(1), query_text,
                               self.pad_val, [l.weight for l in lins], [l.bias for l in lins], self.cq_linear.weight,
                               self.cq_linear.bias, self.ca_linear.weight.view(-1), self.ca_linear.bias)
        self.relational_ins = ins[:, I - 1]
        return ins


class _GraphLayerBase(nn.Module):
    """State shared by the two reasoning layers: the layer-input activation matrix [B*N, Kd] whose first D
    columns hold the node embeddings h and whose remaining columns receive the aggregated neighbour
    messages -- the ``torch.cat`` of reasongnn.py:158-161 / nsm_gnn.py:62 is never materialised by a copy,
    the aggregation kernel writes straight into its slot.  Two storage modes:

      planes (default): the matrix is kept as split-bf16 hi/lo planes (hi + lo = value to 2^-18), which is
          the A-operand layout of the wgmma e2e GEMM; h additionally lives in fp32 ``h32`` [B*N, D].
      fp32: ping-pong fp32 buffers X[2] feeding the exact-fp32 SIMT linear (ops.TC_LINEAR = False)."""

    _plane_cache = {}     # (device, Nt, Kp) -> zero-initialised ping-pong planes, reused across forwards

    def _alloc(self, Nt, Kd, device):
        D = self.entity_dim
        self.use_planes = ops.tc_planes_ok(D, D)
        self.cur = 0
        self.Kd = Kd
        if self.use_planes:
            # every segment ([h | nb_0 | nb_1 ...], D columns each) starts on a 32-byte sector: pitch = D rounded
            # up to 16 bf16 columns (a 32-byte-sector-aligned segment start keeps the plane writes whole sectors);
            # padding columns stay zero forever (nothing writes them), so the padded GEMM is exact
            self.Dp = (D + 15) // 16 * 16
            self.Kpad = Kd // D * self.Dp
            Kp = (self.Kpad + 63) // 64 * 64    # 128-byte row pitch: every TMA-stored piece is sector aligned
            key = (str(device), Nt, Kp, D)
            if key not in _GraphLayerBase._plane_cache:
                _GraphLayerBase._plane_cache.clear()
                _GraphLayerBase._plane_cache[key] = [
                    [torch.zeros(Nt, Kp, dtype=torch.bfloat16, device=device) for _ in range(2)]
                    for _ in range(2)]
            self.P = _GraphLayerBase._plane_cache[key]
            self.h32 = torch.empty(Nt, D, dtype=torch.float32, device=device)
            self.h32_valid = False
            self.fr_rows = torch.empty(Nt, dtype=torch.int32, device=device)
            self.fr_count = torch.zeros(1, dtype=torch.int32, device=device)
            self.dots = torch.empty(2 * Nt, dtype=torch.float32, device=device)
        else:
            self.X = [torch.empty(Nt, Kd, dtype=torch.float32, device=device) for _ in range(2)]

    @property
    def h_view(self):
        """fp32 node embeddings [B*N, D].  In planes mode the fp32 copy is only written when a consumer asked for
        it (``need_h32``); otherwise it is rebuilt on demand from the hi/lo planes (exact to 2^-18)."""
        if not self.use_planes:
            return self.X[self.cur][:, : self.entity_dim]
        if not self.h32_valid:
            D = self.entity_dim
            hi, lo = self.P[self.cur]
            torch.add(hi[:, :D].float(), lo[:, :D].float(), out=self.h32)
            self.h32_valid = True
        return self.h32

    def cur_planes(self):
        return tuple(self.P[self.cur]) if self.use_planes else None

    def _next_planes(self, next_layer):
        """Output planes of a layer: the next layer's A operand, or None when no layer follows (nothing reads them,
        and ``cur_planes()`` is stale after such a layer)."""
        return tuple(self.P[1 - self.cur]) if next_layer else None

    def _h_out(self, need_h, h_rows):
        """The h a layer returns.  With ``h_rows`` in planes mode it may be ``h32`` written on those rows only
        (``h32_valid`` False): a seed-row view for the query reform, which reads nothing else.  ``h_view`` never
        returns such a copy: it rebuilds h from the planes."""
        if not need_h:
            return None
        if h_rows is not None and self.use_planes and not self.h32_valid:
            return self.h32
        return self.h_view

    def _e2e_and_score(self, e2e, mask, need_h32=True, next_layer=True):
        """h <- relu(e2e([h, nb...])); dist = softmax(score_func(h) + mask).  ``need_h32``: also write the fp32
        copy of h (only the instruction update after the last layer of an iteration reads it); ``next_layer``
        False: no output planes."""
        D = self.entity_dim
        sw, sb = self.score_func.weight.view(-1), self.score_func.bias
        if self.use_planes:
            hi, lo = self.P[self.cur]
            ops.linear_tc_planes(hi, lo, self.Kpad, e2e.weight, e2e.bias, out=self.h32 if need_h32 else None,
                                 out_planes=self._next_planes(next_layer), w_score=sw, dots=self.dots, relu=True,
                                 k_seg=D, k_seg_pitch=self.Dp, single_ok=True)
            self.h32_valid = bool(need_h32)
            self.cur = 1 - self.cur
            return ops.masked_softmax(self.dots, sb, mask, self.B, self.N)
        X, Xn = self.X[self.cur], self.X[1 - self.cur]
        ops.e2e_linear(X, e2e.weight, e2e.bias, Xn[:, :D])
        self.cur = 1 - self.cur
        return ops.score_softmax(self.h_view, sw, sb, mask, self.B, self.N)


class ReasonGNNLayer(_GraphLayerBase):
    def __init__(self, args, num_entity, num_relation, entity_dim, alg):
        super().__init__()
        assert alg == "bfs"                                   # reasongnn.py:33
        self.num_entity, self.num_relation, self.entity_dim = num_entity, num_relation, entity_dim
        self.num_ins, self.num_gnn = args["num_ins"], args["num_gnn"]
        self.use_posemb = args["pos_emb"]
        self.normalized_gnn = args["normalized_gnn"]
        D = entity_dim
        self.score_func = nn.Linear(D, 1)
        self.glob_lin = nn.Linear(D, D)                       # unused in forward, kept for the checkpoint
        self.lin = nn.Linear(2 * D, D)                        # unused in forward
        for i in range(self.num_gnn):
            self.add_module("rel_linear" + str(i), nn.Linear(D, D))
            self.add_module("e2e_linear" + str(i), nn.Linear(2 * self.num_ins * D + D, D))
            if self.use_posemb:
                self.add_module("pos_emb" + str(i), nn.Embedding(num_relation, D))
                self.add_module("pos_emb_inv" + str(i), nn.Embedding(num_relation, D))
        self.lin_m = nn.Linear(self.num_ins * D, D)           # unused in forward
        self.linear_drop_train = nn.Dropout(p=args.get("linear_dropout", 0.0))   # reasongnn.py:34-35 (training path)

    def init_reason(self, db, rel_features):
        """reasongnn.py:46-58.  Also builds the hoisted per-layer relation tables
        P_k = rel_linear_k(rel_features) (+ pos_emb_k): ONE GEMM per layer over the stacked forward/inverse
        relation rows per forward, instead of one Linear over F gathered rows per (iteration, layer,
        instruction, direction)."""
        D = self.entity_dim
        self.graph = db.graph
        self.B, self.N = db.B, db.N
        self.local_entity_mask = (db.local_entity != self.num_entity).float().view(-1)
        self._alloc(db.B * db.N, (2 * self.num_ins + 1) * D, db.local_entity.device)
        self.tables = []
        for k in range(self.num_gnn):
            lin = getattr(self, "rel_linear" + str(k))
            add = None
            if self.use_posemb:
                add = [getattr(self, "pos_emb" + str(k)).weight, getattr(self, "pos_emb_inv" + str(k)).weight]
            tf, ti = ops.rel_table(rel_features, lin.weight, lin.bias, addends=add)
            pn = None
            if self.use_planes and ops.aggregate_dual_abs_supported(db.N, D, self.Dp, tf.shape[0]):
                # tf / ti are the two halves of one stacked [2*R1, D] matrix: one conversion launch for both
                pn_all = ops.pad_table256(tf._base if tf._base is not None else torch.cat([tf, ti]))
                pn = (pn_all[: tf.shape[0]], pn_all[tf.shape[0]:])
            self.tables.append((tf, ti, pn))

    def _forward_sparse_prior(self, current_dist, relational_ins, step, need_h):
        """Layer whose prior is non-zero on few nodes (csrc/frontier.cu): GEMM over the h segment only for
        every row, exact recomputation of the frontier rows."""
        D = self.entity_dim
        g = self.graph
        tf, ti, _pn = self.tables[step]
        wt, wh = (g.w_t, g.w_h) if self.normalized_gnn else (None, None)
        e2e = getattr(self, "e2e_linear" + str(step))
        sw, sb = self.score_func.weight.view(-1), self.score_func.bias
        cur, nxt = tuple(self.P[self.cur]), tuple(self.P[1 - self.cur])
        ops.frontier_rows(g, current_dist, self.fr_rows, self.fr_count)
        ops.linear_tc_planes(cur[0], cur[1], self.Dp, e2e.weight[:, :D], e2e.bias,
                             out=self.h32 if need_h else None, out_planes=nxt, w_score=sw, dots=self.dots,
                             relu=True, k_seg=D, k_seg_pitch=self.Dp)
        ops.frontier_fixup(g, current_dist, tf, ti, relational_ins, cur, e2e.weight, e2e.bias, sw, nxt,
                           self.h32 if need_h else None, self.dots, self.fr_rows, self.fr_count, wt, wh)
        self.h32_valid = bool(need_h)
        self.cur = 1 - self.cur
        dist = ops.masked_softmax(self.dots, sb, self.local_entity_mask, self.B, self.N)
        return dist, (self.h_view if need_h else None)

    def forward(self, current_dist, relational_ins, step=0, need_h=True, sparse_prior=False, h_rows=None,
                next_layer=True):
        """One GNN layer (reasongnn.py:134-174): aggregate both directions for every instruction into the
        concat slots, h <- relu(e2e_k([h, nb...])), score, masked softmax.  Returns (dist, h) with h = None when
        ``need_h`` is False (the caller does not read the embeddings of this layer).
        ``h_rows`` (fp32 [B*N], e.g. ``query_entities``): the caller reads only the rows of h with h_rows != 0, and
        the grouped-order dense layer (:func:`ops.dense_layer`) writes no other row of ``h32`` (:meth:`_h_out`); the
        other paths write every row.  ``next_layer`` False: no layer runs after this one in the forward, so the
        dense-prior GEMM writes no operand planes for it; the sparse-prior path writes them all the same."""
        assert next_layer or (need_h and h_rows is None), "a last layer keeps the full fp32 h"
        D = self.entity_dim
        g = self.graph
        if sparse_prior and self.use_planes and ops.SPARSE_PRIOR_FASTPATH:
            return self._forward_sparse_prior(current_dist, relational_ins, step, need_h)
        tf, ti, pn = self.tables[step]
        wt, wh = (g.w_t, g.w_h) if self.normalized_gnn else (None, None)
        e2e = getattr(self, "e2e_linear" + str(step))
        if (self.use_planes and pn is not None and ops.AGG_ABS and ops.FUSED_LAYER and not ops.ACT_BF16
                and self.B * self.N >= ops.FUSED_MIN_ROWS and ops.fused_layer_supported(self.N, D, self.Dp, self.num_ins, D)):
            # the dense layer in grouped K order: one fused kernel, or the aggregation kernel + the full-width GEMM
            sw, sb = self.score_func.weight.view(-1), self.score_func.bias
            ops.dense_layer(g, current_dist, pn[0], pn[1], relational_ins, self.cur_planes(), self.Dp, e2e.weight,
                            e2e.bias, out=self.h32 if need_h else None, out_planes=self._next_planes(next_layer),
                            w_score=sw, dots=self.dots, w_t=wt, w_h=wh, out_rows=h_rows if need_h else None)
            self.h32_valid = bool(need_h) and h_rows is None
            self.cur = 1 - self.cur
            dist = ops.masked_softmax(self.dots, sb, self.local_entity_mask, self.B, self.N)
            return dist, self._h_out(need_h, h_rows)
        if self.use_planes and pn is not None and ops.AGG_ABS:
            ops.aggregate_dual_abs(g, current_dist, pn[0], pn[1], relational_ins, self.cur_planes(), self.Dp,
                                  self.Dp, wt, wh)
        elif self.use_planes:
            ops.aggregate_dual(g, current_dist, tf, ti, relational_ins, None, self.Dp, wt, wh,
                               planes=self.cur_planes(), seg_pitch=self.Dp)
        else:
            ops.aggregate_dual(g, current_dist, tf, ti, relational_ins, self.X[self.cur], D, wt, wh)
        dist = self._e2e_and_score(getattr(self, "e2e_linear" + str(step)), self.local_entity_mask, need_h, next_layer)
        return dist, self._h_out(need_h, h_rows)


class NSMLayer(_GraphLayerBase):
    def __init__(self, args, num_entity, num_relation, entity_dim):
        super().__init__()
        self.num_entity, self.num_relation, self.entity_dim = num_entity, num_relation, entity_dim
        self.num_steps = args["num_step"]
        self.reason_kb = args["reason_kb"]
        self.normalized_gnn = args["normalized_gnn"]
        D = entity_dim
        self.score_func = nn.Linear(D, 1)
        self.lin = nn.Linear(2 * D, D)                        # unused in forward
        for i in range(self.num_steps):
            self.add_module("rel_linear" + str(i), nn.Linear(D, D))
            self.add_module("e2e_linear" + str(i), nn.Linear(2 * D, D))
        self.linear_drop_train = nn.Dropout(p=args.get("linear_dropout", 0.0))   # nsm_gnn.py:30-31 (training path)

    def init_reason(self, db, rel_features):
        D = self.entity_dim
        self.graph = db.graph
        self.B, self.N = db.B, db.N
        self.local_entity_mask = (db.local_entity != self.num_entity).float().view(-1)
        self._alloc(db.B * db.N, 2 * D, db.local_entity.device)
        self.tables = []
        for k in range(self.num_steps):
            lin = getattr(self, "rel_linear" + str(k))
            self.tables.append(ops.rel_table(rel_features, lin.weight, lin.bias, dirs=1)[0])
        self.possible = torch.empty(db.B * db.N, dtype=torch.float32, device=db.local_entity.device)
        if self.use_planes:
            self.nb32 = torch.empty(db.B * db.N, D, dtype=torch.float32, device=db.local_entity.device)

    def forward(self, current_dist, relational_ins, step=0):
        """nsm_gnn.py:54-77 + :87-112 (forward direction only, e2e: 2D -> D)."""
        D = self.entity_dim
        g = self.graph
        w = g.w_t if self.normalized_gnn else None
        if self.use_planes:
            # single-direction aggregate writes fp32; split into the planes' neighbour slot
            ops.aggregate(g, "fwd", current_dist, self.tables[step], relational_ins.view(self.B, 1, D),
                          out=self.nb32, out_col0=0, seg_stride=D, w=w, possible=self.possible)
            hi, lo = self.P[self.cur]
            ops.split_bf16(self.nb32, hi[:, self.Dp:], lo[:, self.Dp:])
        else:
            ops.aggregate(g, "fwd", current_dist, self.tables[step], relational_ins.view(self.B, 1, D),
                          out=self.X[self.cur], out_col0=D, seg_stride=D, w=w, possible=self.possible)
        mask = self.local_entity_mask * self.possible if self.reason_kb else self.local_entity_mask
        return self._e2e_and_score(getattr(self, "e2e_linear" + str(step)), mask, need_h32=False)


def live_plane_buffers():
    """Strong references to the operand planes the reasoning layers currently cache (held by GraphedStep entries: a
    captured graph reads and writes them, and relies on their zero pad columns, after the cache has moved on)."""
    return [t for cache in (_GraphLayerBase._plane_cache, GraftLayer._plane_cache) for sets in cache.values()
            for pair in sets for t in pair]


class GraftLayer(nn.Module):
    """GraftNet's reasoning layer (graft_gnn.py:14-153): query-conditioned fact attention once per forward, then per
    layer a PageRank step over the graft facts and a node update.  Per layer i, on split-bf16 operand planes with five
    D-column segments at pitch Dp, ``[sum_v | indeg | h | q2e | f2e]``:

      head_tab = kb_head_i(h)                               GEMM over the h segment
      gr_graft_aggregate                                    sum_v, indeg, q2e[b] -> planes; d' -> fp32
      f2e = relu([sum_v | indeg | h] @ [W_tail | b_tail e_0 | W_self]^T + b_self)
                                                            = relu(kb_self(h) + sum_f kb_tail(v_f)): the per-fact bias
                                                              enters as indeg(n) * b_tail through the indeg column
      query_emb = W_e2q (sum_n d' x) + (sum_n d') b_e2q     (not for the last layer: the reference never reads it)
      h <- relu([h | q2e | f2e] @ [W_e2e[:, :2D] | fact_scale W_e2e[:, 2D:]]^T + b); score dot in the epilogue
    """

    K_SEGMENTS = 5
    _plane_cache = {}

    def __init__(self, args, num_entity, num_relation, entity_dim):
        super().__init__()
        self.num_entity, self.num_relation, self.entity_dim = num_entity, num_relation, entity_dim
        self.num_layer = args["num_layer"]
        self.pagerank_lambda = args["pagerank_lambda"]
        self.fact_scale = args["fact_scale"]
        self.k = 3
        D = entity_dim
        self.score_func = nn.Linear(D, 1)
        for i in range(self.num_layer):
            self.add_module("q2e_linear" + str(i), nn.Linear(D, D))
            self.add_module("e2q_linear" + str(i), nn.Linear(self.k * D, D))
            self.add_module("e2e_linear" + str(i), nn.Linear(self.k * D, D))
            self.add_module("kb_head_linear" + str(i), nn.Linear(D, D))
            self.add_module("kb_tail_linear" + str(i), nn.Linear(D, D))
            self.add_module("kb_self_linear" + str(i), nn.Linear(D, D))
        self.linear_drop_train = nn.Dropout(p=args.get("linear_dropout", 0.0))   # graft_gnn.py:32-33 (training path)

    def lin(self, name, i):
        return getattr(self, name + str(i))

    def init_reason(self, db, rel, query_hidden_emb, query_mask):
        """graft_gnn.py:45-61 + compute_attention (:64-87), which the reference runs at step 0.  ``rel``: fp32
        relation features [R1, D]."""
        D = self.entity_dim
        if not ops.tc_planes_ok(D, D):
            raise NotImplementedError("GraftNet runs its GEMMs on the wgmma path: entity_dim must be in [8, %d]"
                                      % ops.TC_MAX_N_SPLIT)
        dev = db.local_entity.device
        self.db, self.gg = db, db.graft
        self.B, self.N = db.B, db.N
        Nt = db.B * db.N
        self.local_entity_mask = (db.local_entity != self.num_entity).float().view(-1)
        self.Dp = (D + 15) // 16 * 16
        Kp = (self.K_SEGMENTS * self.Dp + 63) // 64 * 64
        key = (str(dev), Nt, Kp)
        if key not in GraftLayer._plane_cache:
            GraftLayer._plane_cache.clear()
            GraftLayer._plane_cache[key] = [[torch.zeros(Nt, Kp, dtype=torch.bfloat16, device=dev) for _ in range(2)]
                                            for _ in range(2)]
        self.P = GraftLayer._plane_cache[key]
        self.cur = 0
        f32 = dict(dtype=torch.float32, device=dev)
        self.h32 = torch.empty(Nt, D, **f32)
        self.f2e32 = torch.empty(Nt, D, **f32)
        self.head_tab = torch.empty(Nt, D, **f32)
        self.dots = torch.empty(2 * Nt, **f32)
        self.self_tabs = [ops.rel_linear(rel, self.lin("kb_self_linear", i).weight, self.lin("kb_self_linear", i).bias)
                          for i in range(self.num_layer)]
        _w, self.W_tilde, self.E = ops.graft_attention(self.gg, query_hidden_emb, query_mask, rel)

    def seg(self, planes, k, width=None):
        c0 = k * self.Dp
        c1 = c0 + (self.entity_dim if width is None else width)
        return planes[0][:, c0:c1], planes[1][:, c0:c1]

    def h_planes(self):
        """Where the initial node embeddings go (the h segment of the current planes)."""
        return self.seg(self.P[self.cur], 2)

    def forward(self, dist, query_node, step, last):
        """One layer (graft_gnn.py:111-153).  dist: PageRank prior [B, N]; query_node: [B, D] (query_node_emb at step
        0, the previous layer's query_emb after).  Returns (score [B, N], next prior d' [B, N], query_emb or None)."""
        D, Dp, B, N = self.entity_dim, self.Dp, self.B, self.N
        hi, lo = self.P[self.cur]
        e2e, e2q = self.lin("e2e_linear", step), self.lin("e2q_linear", step)
        kh, kt, ks = self.lin("kb_head_linear", step), self.lin("kb_tail_linear", step), self.lin("kb_self_linear", step)
        q2e_l = self.lin("q2e_linear", step)
        ops.linear_tc_planes(hi[:, 2 * Dp:], lo[:, 2 * Dp:], Dp, kh.weight, kh.bias, out=self.head_tab, relu=False,
                             k_seg=D, k_seg_pitch=Dp)
        q2e = ops.linear(query_node.contiguous(), q2e_l.weight, q2e_l.bias)
        d_next = ops.graft_aggregate(self.gg, self.W_tilde, self.E, dist, self.self_tabs[step], self.head_tab,
                                     self.pagerank_lambda, q2e=q2e, planes=(hi, lo), col_sum=0, col_indeg=Dp,
                                     col_q2e=3 * Dp)
        W1 = torch.zeros(D, 3 * D, dtype=torch.float32, device=hi.device)
        W1[:, :D] = kt.weight
        W1[:, D] = kt.bias
        W1[:, 2 * D:] = ks.weight
        f2e_hi, f2e_lo = self.seg((hi, lo), 4, Dp)
        ops.linear_tc_planes(hi, lo, 3 * Dp, W1, ks.bias, out=self.f2e32, out_planes=(f2e_hi, f2e_lo), relu=True,
                             k_seg=D, k_seg_pitch=Dp)
        query_emb = None
        if not last:
            # sum_n d'[n] x[n] with x = [h | q2e[b] | fact_scale f2e], from the layer-input h (graft_gnn.py:138-140)
            mass = d_next.sum(dim=1, keepdim=True)
            sx = torch.cat([ops.seed_retrieve(d_next, self.h32, B, N, D), mass * q2e,
                            self.fact_scale * ops.seed_retrieve(d_next, self.f2e32, B, N, D)], dim=1)
            query_emb = ops.linear(sx, e2q.weight, None)
            query_emb += mass * e2q.bias
        We = torch.cat([e2e.weight[:, :2 * D], self.fact_scale * e2e.weight[:, 2 * D:]], dim=1)
        nhi, nlo = self.P[1 - self.cur]
        ops.linear_tc_planes(hi[:, 2 * Dp:], lo[:, 2 * Dp:], 3 * Dp, We, e2e.bias, out=self.h32,
                             out_planes=self.seg((nhi, nlo), 2), w_score=self.score_func.weight.view(-1),
                             dots=self.dots, relu=True, k_seg=D, k_seg_pitch=Dp)
        self.cur = 1 - self.cur
        score = ops.masked_softmax(self.dots, self.score_func.bias, self.local_entity_mask, B, N)
        return score, d_next, query_emb

    def logits(self):
        """score_func(h) of the last layer, unmasked [B, N] (the loss input, graft_gnn.py:144)."""
        d = self.dots.view(2, -1)
        return (d[0] + d[1] + self.score_func.bias).view(self.B, self.N)
