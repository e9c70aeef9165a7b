"""Run-time defaults of the g2pc host layer (module attributes; change them before calling the drop-in API)."""
import torch

# Base seed of the Philox stream (key); counter = (global Gaussian id, sample, attempt, call id).
SEED = 42

# Accept test of the Mahalanobis cull: 1 = explicit sqrt(d^T Sigma^-1 d) <= std in fp32, as the reference computes
# it (gauss_to_pc.py:92-103); 0 = |eps| <= std (equal in exact arithmetic, cheaper).
CULL_MODE = 1

# dtype of the colour / normal outputs of generate_pointcloud.  The reference returns float64 for both (an artefact
# of torch.cat type promotion, gauss_to_pc.py:317-318,352-369) and casts to u8 / f4 when writing the PLY
# (gauss_dataloader.py:176-200); float32 halves the output traffic and leaves the PLY bytes unchanged.
OUTPUT_DTYPE = torch.float32

# Dense attempts the count pass stores on its first try; if a Gaussian still emits in a later attempt the sampler
# replays the (deterministic) stream with every attempt stored (gauss_to_pc._attempt_ladder).
ATTEMPTS_STORED_FIRST = 16

# python-renderer tile parameters.  The reference derives them from free GPU memory at call time
# (gauss_render.py:440-444), which makes results hardware dependent; they are pinned to render()'s own defaults
# (gauss_render.py:266).
MAX_TILE_SIZE = 60
MAX_GAUSSIANS_PER_TILE = 60000

# Transmittance below which a warp of the blend kernel stops walking its tile's list (all of its 128 pixels must be
# below it).  Every skipped contribution is then < BLEND_T_STOP and so is their sum per pixel, i.e. colours, images and
# per-Gaussian maximum contributions move by less than 1e-6 (the parity contract is 1e-4).  0 selects FLT_MIN: only
# contributions that underflow are dropped (the strict-parity tests use it).  The reference's CUDA back-end stops each
# pixel at T < 1e-4 (forward.cu:415); its python back-end never stops.
BLEND_T_STOP = 1e-6

# Frames (cameras) in flight in the colour stage: 2 = the front-end of camera f + 1 overlaps the blend of camera f on a
# second CUDA stream (g2pc/frames.py); 1 = strictly serial.
FRAME_SLOTS = 2

# python back-end, async mode: consecutive cameras of one resolution projected by one preprocess launch, which reads the
# scene once per batch instead of once per camera (g2pc/frames.py, csrc/s3_preprocess.cu).  1..8; 1 = one launch per
# camera.  Each further camera costs two more sets of per-camera outputs (N x 60 bytes each: 180 MB at 3 M Gaussians).
PREPROCESS_CAMERAS = 4

# NVTX ranges around the stages of the pipeline (covariances / colour stage / culls / validate / sampling) and around
# every camera: visible in nsys / ncu timelines, ~1 us each when no tool is attached.
NVTX = True
