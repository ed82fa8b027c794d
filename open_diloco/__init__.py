"""Import-path compatibility with the reference package: ``open_diloco.hivemind_diloco``, ``open_diloco.utils``,
``open_diloco.ckpt_utils``, ``open_diloco.train_fsdp`` resolve to the H100-native implementations in
``opendiloco_b200`` so code written against PrimeIntellect-ai/OpenDiloco keeps importing."""
