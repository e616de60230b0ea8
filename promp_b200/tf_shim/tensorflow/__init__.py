"""An 8-symbol stand-in for `import tensorflow as tf` so that the reference's UNCHANGED driver
(meta_policy_search/meta_trainer.py:1,55-57,72-76,152) can run on top of promp_b200, whose state lives
on the GPU rather than in a TF session.  Put promp_b200/tf_shim on sys.path *instead of* TensorFlow.
Not used by promp_b200 itself."""


class Session(object):
    def __init__(self, *args, **kwargs):
        self._closed = False

    def as_default(self):
        return self

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False

    def run(self, fetches, feed_dict=None):
        if isinstance(fetches, (list, tuple)):
            return [self.run(f) for f in fetches]
        return fetches() if callable(fetches) else fetches

    def close(self):
        self._closed = True


def global_variables():
    return []            # nothing to initialise: parameters are created initialised on the device


def is_variable_initialized(var):
    return True


def variables_initializer(var_list, name='init'):
    return None


def get_default_session():
    return Session()


def set_random_seed(seed):
    pass


def tanh(x):            # lets run scripts pass hidden_nonlinearity=tf.tanh and output_nonlinearity=tf.tanh
    raise NotImplementedError("symbolic placeholder: promp_b200 policies evaluate tanh in CUDA")


class nn(object):       # tf.nn.relu: lets run scripts pass hidden_nonlinearity=tf.nn.relu
    @staticmethod
    def relu(x):
        raise NotImplementedError("symbolic placeholder: promp_b200 policies evaluate relu in CUDA")
