"""Parameter bags with the reference's field names and defaults (rl_coach/base_parameters.py:181-420,
rl_coach/agents/dqn_agent.py:33-66, rl_coach/core_types.py step types).  Only the fields the replay -> learn path
reads are present; everything is a plain attribute so presets can set them the way Coach presets do."""


class StepMethod(object):
    def __init__(self, num_steps):
        self.num_steps = int(num_steps)


class EnvironmentSteps(StepMethod):
    pass


class TrainingSteps(StepMethod):
    pass


class EnvironmentEpisodes(StepMethod):
    pass


class MiddlewareScheme(object):
    """rl_coach/base_parameters.py:44-48; FC middleware layer lists of
    architectures/tensorflow_components/middlewares/fc_middleware.py:56-80"""
    Empty = "Empty"
    Shallow = "Shallow"
    Medium = "Medium"
    Deep = "Deep"
    units = {"Empty": (), "Shallow": (64,), "Medium": (512,), "Deep": (128, 128, 128)}


class MiddlewareParameters(object):
    def __init__(self, scheme=MiddlewareScheme.Medium):
        self.scheme = scheme        # a MiddlewareScheme name or a list of Dense specs (fc_middleware.py:56-80)


class InputEmbedderParameters(object):
    """architectures/embedder_parameters.py: scheme "Medium" (the default embedders) or a list of Conv2d / Dense specs"""

    def __init__(self, scheme="Medium"):
        self.scheme = scheme


class Conv2d(object):
    """architectures/layers.py Conv2d(num_filters, kernel_size, strides): one VALID, ReLU convolution of a scheme"""

    def __init__(self, num_filters, kernel_size, strides):
        self.num_filters, self.kernel_size, self.strides = int(num_filters), int(kernel_size), int(strides)


class Dense(object):
    """architectures/layers.py Dense(units): one ReLU dense layer of a scheme"""

    def __init__(self, units):
        self.units = int(units)


def scheme_layers(scheme):
    """an embedder scheme as QNetworkDef's embedder_scheme: None for the Medium default, else the list of specs"""
    if isinstance(scheme, (list, tuple)):
        return list(scheme)
    if getattr(scheme, "value", scheme) != "Medium":
        raise ValueError("embedder scheme %r: only Medium or an explicit layer list is implemented" % (scheme,))
    return None


def middleware_units(scheme):
    """a middleware scheme as QNetworkDef's middleware_units"""
    if isinstance(scheme, (list, tuple)):
        return tuple(d.units for d in scheme)
    return MiddlewareScheme.units[getattr(scheme, "value", scheme)]


class AlgorithmParameters(object):
    def __init__(self):
        self.num_consecutive_playing_steps = EnvironmentSteps(1)
        self.num_consecutive_training_steps = 1
        self.discount = 0.99
        self.num_steps_between_copying_online_weights_to_target = TrainingSteps(0)
        self.rate_for_copying_weights_to_target = 1.0
        self.n_step = -1
        self.update_pre_network_filters_state_on_train = False
        self.update_pre_network_filters_state_on_inference = True


class NetworkParameters(object):
    def __init__(self):
        self.clip_gradients = None
        self.gradients_clipping_method = "ClipByGlobalNorm"
        self.l2_regularization = 0
        self.learning_rate = 0.00025
        self.optimizer_type = 'Adam'
        self.optimizer_epsilon = 0.0001
        self.adam_optimizer_beta1 = 0.9
        self.adam_optimizer_beta2 = 0.99
        self.batch_size = 32
        self.replace_mse_with_huber_loss = False
        self.create_target_network = False
        self.scale_down_gradients_by_number_of_workers_for_sync_training = True
        self.middleware_parameters = MiddlewareParameters()


class AgentParameters(object):
    def __init__(self, algorithm, memory, networks):
        self.algorithm = algorithm
        self.memory = memory
        self.network_wrappers = networks
        self.input_filter = None
        self.pre_network_filter = None
        self.is_batch_rl_training = False
