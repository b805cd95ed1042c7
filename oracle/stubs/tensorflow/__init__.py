"""Empty stand-in for tensorflow: NonlinearPositionController.__init__ (quadrotor_control.py:256) imports it even with
tf_control=False, the only setting QuadrotorEnvMulti passes, and never uses it then."""
