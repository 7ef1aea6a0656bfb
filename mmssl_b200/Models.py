"""Drop-in replacement for the reference's ``Models.py`` (HKUDS/MMSSL, MMSSL/Models.py).

``from Models import MMSSL, Discriminator`` (main.py:27) keeps working: same constructor and
``forward`` signatures, same registered parameter names (state_dict compatible), same module-global
``args`` convention (Models.py:13-15), same 12-tuple with outputs 0/6 and 1/7 being the same objects
(Models.py:220).  What changes is what runs: ``forward`` is ONE autograd node whose forward and
backward are the sm_90a kernels of libmmssl_b200 (functional.MMSSLForwardFn) -- CSR SpMM with fused
softmax / layer-sum epilogues, wgmma projection, fused row-wise glue.  There is no eager fallback.

``Discriminator`` stays a stock-torch module with the reference's architecture so that the reference's own trainer and its
checkpoints keep working; the device implementation of the GAN side (no autograd) is mmssl_b200/gan.py + fullstep.py, which
reads and updates this module's state_dict in place (mmssl_b200/trainer.py).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

try:                                    # inside the reference tree: the reference's own flags
    from utility.parser import parse_args
    args = parse_args()
except Exception:                       # stand-alone use: same defaults (mmssl_b200/config.py)
    from mmssl_b200.config import default_args
    args = default_args()

from mmssl_b200.engine import Engine, FeatureStore
from mmssl_b200.functional import MMSSLForwardFn, batched_contrastive_loss as _nce
from mmssl_b200.graph import prepare


class MMSSL(nn.Module):
    def __init__(self, n_users, n_items, embedding_dim, weight_size, dropout_list, image_feats, text_feats,
                 register_feature_embeddings: bool = True, proj_impl: str = "tc"):
        super().__init__()
        d = args.embed_size
        self.n_users, self.n_items, self.embedding_dim = n_users, n_items, embedding_dim
        self.n_ui_layers = len(weight_size)
        self.weight_size = [embedding_dim] + list(weight_size)
        dv, dt = image_feats.shape[1], text_feats.shape[1]

        # Parameter creation order follows the reference (Models.py:28-66) so that a seeded
        # construction draws the same initial values from torch's global RNG.
        self.image_trans = nn.Linear(dv, d)
        self.text_trans = nn.Linear(dt, d)
        for lin in (self.image_trans, self.text_trans):
            nn.init.xavier_uniform_(lin.weight)
        self.encoder = nn.ModuleDict({"image_encoder": self.image_trans, "text_encoder": self.text_trans})
        self.common_trans = nn.Linear(d, d)                     # registered, unused by forward (SURVEY B.2)
        nn.init.xavier_uniform_(self.common_trans.weight)
        self.align = nn.ModuleDict({"common_trans": self.common_trans})
        self.user_id_embedding = nn.Embedding(n_users, embedding_dim)
        self.item_id_embedding = nn.Embedding(n_items, embedding_dim)
        for emb in (self.user_id_embedding, self.item_id_embedding):
            nn.init.xavier_uniform_(emb.weight)

        dev = torch.device("cuda")
        img = torch.as_tensor(np.asarray(image_feats)).float()
        txt = torch.as_tensor(np.asarray(text_feats)).float()
        self.image_feats = img.to(dev)          # plain constant tensors, as in Models.py:46-47
        self.text_feats = txt.to(dev)
        if register_feature_embeddings:         # I x D trainable copies the reference registers but never uses
            self.image_embedding = nn.Embedding.from_pretrained(img, freeze=False)
            self.text_embedding = nn.Embedding.from_pretrained(txt, freeze=False)

        self.softmax = nn.Softmax(dim=-1)
        self.act = nn.Sigmoid()
        self.sigmoid = nn.Sigmoid()
        self.dropout = nn.Dropout(p=args.drop_rate)
        self.batch_norm = nn.BatchNorm1d(d)
        self.tau = 0.5
        names = ("w_q", "w_k", "w_v", "w_self_attention_item", "w_self_attention_user")
        wd = {k: nn.Parameter(nn.init.xavier_uniform_(torch.empty(d, d))) for k in names}
        wd["w_self_attention_cat"] = nn.Parameter(nn.init.xavier_uniform_(torch.empty(args.head_num * d, d)))
        self.weight_dict = nn.ParameterDict(wd)
        self.embedding_dict = {"user": {}, "item": {}}

        self._engine = Engine(d, self.n_ui_layers, head_num=args.head_num, id_cat_rate=args.id_cat_rate,
                              model_cat_rate=args.model_cat_rate, proj_impl=proj_impl)
        self._feats = None          # FeatureStore pair, built lazily on the parameters' device

    # ------------------------------------------------------------------ reference helper API
    def mm(self, x, y):
        """Models.py:69-73 -- the SpMM plug point, now the CUDA operator."""
        from mmssl_b200.functional import spmm
        return spmm(x, y)

    def batched_contrastive_loss(self, z1, z2, batch_size=4096):
        """Models.py:79-98 (tau = self.tau, no +1e-8; unused by the reference trainer)."""
        raise NotImplementedError("the trainer-side loss is mmssl_b200.functional.batched_contrastive_loss "
                                  "(main.py:218-249); Models.py:79-98 is dead code in the reference")

    # ------------------------------------------------------------------ forward
    def _feature_stores(self):
        if self._feats is None:
            keep = self._engine.proj_impl != "tc"
            self._feats = (FeatureStore(self.image_feats, keep_fp32=True), FeatureStore(self.text_feats, keep_fp32=True))
            del keep
        return self._feats

    def forward(self, ui_graph, iu_graph, image_ui_graph, image_iu_graph, text_ui_graph, text_iu_graph):
        graphs = tuple(prepare(g) for g in (ui_graph, iu_graph, image_ui_graph, image_iu_graph, text_ui_graph, text_iu_graph))
        masks = None
        if self.training and (not isinstance(self.dropout, nn.Dropout) or self.dropout.p > 0):
            # Run the dropout module on ones: same RNG consumption (two [I, d] draws, image first) as
            # the reference's self.dropout(self.image_trans(...)), self.dropout(self.text_trans(...))
            ones = torch.ones(self.n_items, args.embed_size, dtype=torch.float32, device=self.image_feats.device)
            masks = (self.dropout(ones), self.dropout(ones))
        w = self.weight_dict
        o = MMSSLForwardFn.apply(self._engine, self._feature_stores(), graphs, masks,
                                 self.image_trans.weight, self.image_trans.bias, self.text_trans.weight,
                                 self.text_trans.bias, self.user_id_embedding.weight, self.item_id_embedding.weight,
                                 w["w_self_attention_cat"])
        u_f, i_f, i_v, i_t, u_v, u_t, u_vid, u_tid, i_vid, i_tid = o
        self.embedding_dict["user"]["image"], self.embedding_dict["user"]["text"] = u_vid, u_tid
        self.embedding_dict["item"]["image"], self.embedding_dict["item"]["text"] = i_vid, i_tid
        return u_f, i_f, i_v, i_t, u_v, u_t, u_f, i_f, u_vid, u_tid, i_vid, i_tid


class Discriminator(nn.Module):
    """GAN discriminator of the reference (Models.py:224-245), stock torch (parameter container for fullstep.FullStep).
    ``nn.LeakyReLU(True)`` means negative_slope == 1.0, i.e. identity (SURVEY B.7) -- kept as is."""

    def __init__(self, dim):
        super().__init__()
        h1, h2 = int(dim / 4), int(dim / 8)
        self.net = nn.Sequential(
            nn.Linear(dim, h1), nn.LeakyReLU(True), nn.BatchNorm1d(h1), nn.Dropout(args.G_drop1),
            nn.Linear(h1, h2), nn.LeakyReLU(True), nn.BatchNorm1d(h2), nn.Dropout(args.G_drop2),
            nn.Linear(h2, 1), nn.Sigmoid())

    def forward(self, x):
        return (100 * self.net(x.float())).view(-1)
