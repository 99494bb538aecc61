"""b200mvs: the dense MVS depth-map hot path of MVE (libs/dmrecon) on H100.

`mve_b200.dmrecon`  - Settings / Scene / DMRecon over the C ABI of libb200mvs.so (include/b200mvs.h)
`mve_b200.sharding` - reference views over ranks, all-gather of the input images
`mve_b200.synth`    - synthetic scenes of the BASELINE configs, MVE scene directory writer
`mve_b200.build`    - nvcc build of the library (sm_90a)
"""
__version__ = "0.1"
