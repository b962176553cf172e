"""Data pipeline: ES-futures time-series windowing/scaling (reference parity) + synthetic generators."""
from .timeseries import (x_cols, y_cols, read_file_from_aws, reshape_and_scale_data_for_training,
                         TimeSeriesDataSet, MinMaxScaler, StandardScaler,
                         synthetic_market_frame, ensure_dataset)  # noqa: F401
from .synthetic import SyntheticImageBatches, SyntheticTokenBatches, DeviceBatchLoader  # noqa: F401
