"""graphsage_b200 - an H100-native (sm_90a) sample-and-aggregate engine behind the
graphsage.neigh_samplers / graphsage.aggregators / graphsage.models.SampleAndAggregate surface of
williamleif/GraphSAGE.  `import graphsage_b200 as graphsage` is the intended drop-in for that path.

All compute goes through libgraphsage_b200.so (include/graphsage_b200.h); there is no CPU fallback.
"""
from . import (_lib, aggregators, graph, graphed_training, host_features, inits, int8_features, layers, minibatch,  # noqa: F401
               models, neigh_samplers, node2vec, ops, prediction, utils)
from .aggregators import (GCNAggregator, MaxPoolingAggregator, MeanAggregator, MeanPoolingAggregator,  # noqa: F401
                          SeqAggregator, TwoMaxLayerPoolingAggregator, set_default_math)
from .graphed_training import GraphedTrainStep, make_adam_capturable  # noqa: F401
from .host_features import HostFeatures  # noqa: F401
from .int8_features import Int8Features  # noqa: F401
from .layers import Dense, Layer, identity, relu  # noqa: F401
from .models import Node2VecModel, SAGEInfo, SampleAndAggregate  # noqa: F401
from .neigh_samplers import CSRNeighborSampler, UniformNeighborSampler  # noqa: F401
from .prediction import BipartiteEdgePredLayer  # noqa: F401
from .supervised_models import SupervisedGraphsage  # noqa: F401
from .unsupervised_models import UnigramNegativeSampler, UnsupervisedGraphsage  # noqa: F401

__version__ = "0.1.0"
