"""Thin runner with the reference's contract (rl_x/runner/runner.py:37-384): pre-parse `--algorithm.name / --environment.name /
--runner.mode`, import the plugin packages (which register themselves), check compatibility, build the three config trees
from the plugins' defaults + `--tree.key=value` flags, create envs, construct the model, call train()/test().

absl / ml_collections / gymnasium are not in this image, so flags are parsed by rl_x_b200.config_dict.apply_overrides.
`implementation_package_names` works as in the reference: packages are tried in order, so
`Runner(implementation_package_names=["rl_x_b200", "rl_x"])` lets this package's plugins and reference plugins coexist."""
import importlib
import logging
import logging.handlers
import os
import sys

from rl_x_b200.config_dict import ConfigDict, apply_overrides
from rl_x_b200.runner.runner_mode import RunnerMode
from rl_x_b200.runner.default_config import get_config as get_runner_config
from rl_x_b200.algorithms.algorithm_manager import get_algorithm_config, get_algorithm_model_class, get_algorithm_general_properties
from rl_x_b200.environments.environment_manager import (get_environment_config, get_environment_create_train_and_eval_env,
                                                          get_environment_general_properties)

DEFAULT_ALGORITHM = "ppo.b200"
DEFAULT_ENVIRONMENT = "synthetic.box"
DEFAULT_RUNNER_MODE = "train"

rlx_logger = logging.getLogger("rl_x")


def _names(members):
    return [getattr(m, "name", m) for m in members]


class Runner:
    def __init__(self, implementation_package_names=["rl_x_b200"], argv=None):
        self._argv = list(sys.argv[1:] if argv is None else argv)
        algorithm_name, environment_name, self._mode = self.parse_arguments()

        self.import_environment(environment_name, implementation_package_names)
        environment_general_properties = get_environment_general_properties(environment_name)
        self.import_algorithm(algorithm_name, implementation_package_names)
        algorithm_general_properties = get_algorithm_general_properties(algorithm_name)

        # Compatibility check (runner.py:86-91); enum classes may come from different packages, so compare by member name
        e, a = environment_general_properties, algorithm_general_properties
        if e.action_space_type.name not in _names(a.action_space_types):
            raise ValueError(f"Incompatible action space type. Environment: {e.action_space_type}, Algorithm: {a.action_space_types}")
        if e.observation_space_type.name not in _names(a.observation_space_types):
            raise ValueError(f"Incompatible observation space type. Environment: {e.observation_space_type}, Algorithm: {a.observation_space_types}")
        if e.data_interface_type.name not in _names(a.data_interface_types):
            raise ValueError(f"Incompatible data interface type. Environment: {e.data_interface_type}, Algorithm: {a.data_interface_types}")

        self._config = ConfigDict()
        self._config.runner = get_runner_config(self._mode)
        self._config.algorithm = get_algorithm_config(algorithm_name)
        self._config.environment = get_environment_config(environment_name)
        self._explicitly_set = apply_overrides(self._config, self._argv)

        # torch-interface envs must live on the algorithm's device (runner.py:116-128)
        if e.data_interface_type.name == "TORCH" and "device" in self._config.environment:
            if self._config.algorithm.device != self._config.environment.device:
                raise ValueError("Algorithm and environment device must match for torch-interface environments.")

        self._model_class = get_algorithm_model_class(algorithm_name)
        self._create_train_and_eval_env = get_environment_create_train_and_eval_env(environment_name)

        rlx_logger.setLevel(logging.INFO)
        rlx_logger.propagate = False
        if not rlx_logger.handlers:
            handler = logging.StreamHandler(sys.stdout)
            handler.setFormatter(logging.Formatter("[%(asctime)s] [%(filename)s:%(lineno)d] %(levelname)s - %(message)s", "%m-%d %H:%M:%S"))
            rlx_logger.addHandler(handler)

    def parse_arguments(self):
        def pop(prefix, default):
            hits = [a for a in self._argv if a.startswith(prefix)]
            if not hits:
                return default
            self._argv.remove(hits[0])
            return hits[0].split("=", 1)[1]

        return (pop("--algorithm.name=", DEFAULT_ALGORITHM), pop("--environment.name=", DEFAULT_ENVIRONMENT),
                pop("--runner.mode=", DEFAULT_RUNNER_MODE))

    @staticmethod
    def _import_first(kind, name, implementation_package_names):
        for package in implementation_package_names:
            try:
                importlib.import_module(f"{package}.{kind}.{name}")
                return
            except ModuleNotFoundError as e:
                if e.name is None or not f"{package}.{kind}.{name}".startswith(e.name):
                    raise  # a dependency of an existing plugin is missing: do not hide it
        raise ModuleNotFoundError(f"no implementation package provides {kind}.{name} (searched {implementation_package_names})")

    def import_environment(self, environment_name, implementation_package_names):
        self._import_first("environments", environment_name, implementation_package_names)

    def import_algorithm(self, algorithm_name, implementation_package_names):
        self._import_first("algorithms", algorithm_name, implementation_package_names)

    def run(self):
        if self._mode == RunnerMode.SHOW_CONFIG:
            return self._show_config()
        if self._mode == RunnerMode.TRAIN:
            return self._train()
        if self._mode == RunnerMode.TEST:
            return self._test()
        raise ValueError("Invalid mode")

    def _show_config(self):
        import json
        rlx_logger.info("\n" + json.dumps(self._config.to_dict(), indent=2, default=str))

    def _run_path(self):
        r = self._config.runner
        return os.path.abspath(f"runs/{r.project_name}/{r.exp_name}/{r.run_name}")

    def _build_model(self, run_path, writer):
        train_env, eval_env = self._create_train_and_eval_env(self._config)
        if self._config.runner.load_model:
            explicitly_set = [p for p in self._explicitly_set if p.startswith("algorithm.")]
            model = self._model_class.load(self._config, train_env, eval_env, run_path, writer, explicitly_set)
        else:
            model = self._model_class(self._config, train_env, eval_env, run_path, writer)
        return model, train_env, eval_env

    def _train(self):
        run_path = self._run_path()
        r = self._config.runner
        if r.save_model or r.track_tb or r.track_wandb:
            os.makedirs(run_path, exist_ok=True)
        if r.track_wandb:
            import wandb
            wandb.init(entity=r.wandb_entity, project=r.project_name, group=r.exp_name, name=r.run_name, notes=r.notes,
                       sync_tensorboard=False, config=self._config.to_dict(), save_code=True)
            wandb.define_metric("*", step_metric="global_step")
        writer = None
        if r.track_tb:
            from torch.utils.tensorboard import SummaryWriter
            writer = SummaryWriter(run_path)
            items = list(self._config.runner.items()) + list(self._config.algorithm.items()) + list(self._config.environment.items())
            writer.add_text("hyperparameters", "|param|value|\n|-|-|\n%s" % ("\n".join([f"|{k}|{v}|" for k, v in items])))

        model, train_env, eval_env = self._build_model(run_path, writer)
        self.model = model
        try:
            model.train()
        except Exception:
            rlx_logger.error("Uncaught exception", exc_info=True)  # logged and swallowed like runner.py:340-343
            self.failed = True
        finally:
            train_env.close()
            eval_env.close()
            if r.track_tb:
                writer.close()
            if r.track_wandb:
                import wandb
                wandb.finish()

    def _test(self):
        r = self._config.runner
        if r.track_wandb:
            raise ValueError("Wandb is not supported in test mode")
        if r.track_tb:
            raise ValueError("Tensorboard is not supported in test mode")
        if r.save_model:
            raise ValueError("Saving model is not supported in test mode")
        model, train_env, eval_env = self._build_model(self._run_path(), None)
        try:
            model.test(r.nr_test_episodes)
        except Exception:
            rlx_logger.error("Uncaught exception", exc_info=True)
        finally:
            train_env.close()
            eval_env.close()
