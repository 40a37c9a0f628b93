"""gnn_rag_b200 -- H100-native (sm_90a) implementation of GNN-RAG's GNN retrieval hot path.

Public surface mirrors the reference (cmavro/GNN-RAG ``gnn/``):
    from gnn_rag_b200 import ReaRev, NSM, GraftNet, Evaluator
"""
from .models import NSM, GraftNet, ReaRev  # noqa: F401
from .evaluate import Evaluator, retrieve  # noqa: F401
from .graphed import GraphedGraftTrainStep, GraphedStep, GraphedTrainStep, Sweep  # noqa: F401

__all__ = ["ReaRev", "NSM", "GraftNet", "Evaluator", "retrieve", "GraphedStep", "GraphedTrainStep",
           "GraphedGraftTrainStep", "Sweep"]
