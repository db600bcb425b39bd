"""NeatConfig mirror (utils/neat_config.py:19-119): same YAML files, same sections, same error behaviour.

The TPU RunConfig part (utils/neat_config.py:122-151) has no meaning on a GPU and is dropped; `device.*` TPU keys are
accepted and ignored.  File globs in `data.*_file` are expanded with the stdlib instead of tf.io.gfile.
"""
from __future__ import annotations

import argparse
import glob
import os
from copy import deepcopy

import yaml


class NeatConfig(object):
    def __init__(self):
        self.data = {}
        self.model = {}
        self.optimizer = {}
        self.device = {}
        self.downstream = {}
        self.validate = {}
        self.misc = {}

    @classmethod
    def from_yaml(cls, config_file):
        """utils/neat_config.py:31-43."""
        with open(config_file, "r") as f:
            config_dict = yaml.load(f, Loader=yaml.FullLoader)
        return cls.from_dict(config_dict, orig_config_file=config_file)

    @classmethod
    def from_dict(cls, config_dict, orig_config_file=None):
        """utils/neat_config.py:45-102."""
        config = deepcopy(config_dict)
        if "misc" not in config:
            config["misc"] = {}
        for key in ["data", "model", "optimizer", "device"]:  # mandatory keys, :55-57
            if key not in config:
                raise ValueError("Configuration file {} is missing {}".format(orig_config_file, key))
        if "output_dir" not in config["device"]:  # :60-61
            raise ValueError("Missing output directory")
        for x in ["train_file", "val_file", "test_file"]:  # glob expansion, :72-97
            if x in config["data"]:
                v_list = []
                for input_pattern in config["data"][x].split(","):
                    v_list.extend(sorted(glob.glob(input_pattern)))
                config["data"][f"{x}_expanded"] = v_list
        config_cls = cls()
        config_cls.__dict__.update(config)
        return config_cls

    @classmethod
    def from_args(cls, help_message="NeatConfig", default_config_file=None, argv=None):
        """utils/neat_config.py:104-119."""
        parser = argparse.ArgumentParser(description=help_message)
        parser.add_argument("config_file", nargs="?", help="Where the config.yaml is located",
                            default=default_config_file, type=str)
        args = parser.parse_args(argv)
        if not args.config_file:
            raise ValueError("No config file provided!")
        if not os.path.exists(args.config_file):
            raise ValueError("Config file {} not found?".format(args.config_file))
        return cls.from_yaml(args.config_file)


def patch_embed_variant(model_config: dict) -> dict:
    """Return a copy of a `model:` section with the hybrid ResNet stem switched off (resnet_layers: []), i.e. the
    16x16 patch-embed path of utils/vision_transformer.py:194-205 that BASELINE.json's north star names.
    merlot.yaml as shipped selects the hybrid stem (SURVEY.md discrepancy 1); that path (K13, csrc/stem.cu) runs forward and
    backward as well -- this switch only names the variant the headline benchmark measures."""
    c = deepcopy(model_config)
    c["resnet_layers"] = []
    return c
