from .base_rbm import *
from .rbm import *
from .class_rbm import *
from .group import *
