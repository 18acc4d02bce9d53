"""GPU-side input pipeline (SURVEY.md section 8 row f2): Resize -> [ColorJitter] -> ToTensor -> Normalize with the
MF / MFOnline tuple gather, on uint8 frames resident in device memory; DeviceDataset / DeviceLoader keep a whole
training set resized in device memory and assemble each batch on the GPU in the reference DataLoader's order."""
from .preprocess import ImagePipeline, ColorJitterSampler, resize_output_size  # noqa: F401
from .loader import ItemLayout, DeviceDataset, DeviceLoader, host_batches  # noqa: F401
from . import tuples  # noqa: F401
