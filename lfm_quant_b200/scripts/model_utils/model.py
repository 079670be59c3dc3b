"""Model factory -- the plugin boundary (reference: scripts/model_utils/model.py:14-39): ``nn_type`` is resolved
to a class by name in this module's globals; ``Cls(config, dataset).model`` is returned."""
from __future__ import absolute_import, division, print_function

# All models should be imported here
from ..models.point_estimate.mlp_linear_point_estimate import MLPLinearPointEstimate  # noqa: F401
from ..models.point_estimate.naive_point_estimate import NaivePointEstimate  # noqa: F401
from ..models.point_estimate.rnn_point_estimate import RNNPointEstimate  # noqa: F401
from ..models.uq_range_estimate.rnn_uq_range_estimate import RNNUqRangeEstimate  # noqa: F401

# the hidden-layer MLPs (Dense -> BatchNormalization -> ReLU -> Dropout stacks)
_NOT_BUILT = ('MLPPointEstimate', 'MLPUqRangeEstimate')


class Model(object):

    def __init__(self, config, dataset):
        self._config = config
        self._dataset = dataset

    def get_model(self):
        all_objects = globals()
        if self._config.nn_type in all_objects:
            model_constructor = all_objects[self._config.nn_type]
        elif self._config.nn_type in _NOT_BUILT:
            raise NotImplementedError("nn_type = %s: the hidden-layer MLP models are not built" % self._config.nn_type)
        else:
            raise RuntimeError("Unknown nn_type = %s" % self._config.nn_type)
        m = model_constructor(self._config, self._dataset)
        model = m.model
        print(model.summary())
        if self._config.UQ:
            assert 'uq' in self._config.nn_type.lower(), "UQ should be True only for UQ Models"
        else:
            assert 'point' in self._config.nn_type.lower(), "UQ should be False for Point Estimate Models"
        return model
