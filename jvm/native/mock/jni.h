/* Minimal stand-in for <jni.h>: ONLY for `gcc -fsyntax-only` of jvm/native/snappy_gpu_jni.c in a container without a
 * JDK (tests/test_jni_syntax.py).  It declares the JNIEnv function-table members the shim uses with the signatures of
 * the JNI specification (Java SE 8, "JNI Functions"); the member ORDER of the real table is irrelevant for a syntax and
 * type check.  Never ship or link against this file. */
#ifndef MOCK_JNI_H
#define MOCK_JNI_H
#include <stdint.h>

typedef int32_t jint;
typedef int64_t jlong;
typedef int8_t jbyte;
typedef double jdouble;
typedef uint8_t jboolean;
typedef jint jsize;
struct _jobject;
typedef struct _jobject* jobject;
typedef jobject jclass;
typedef jobject jarray;
typedef jarray jobjectArray;
typedef jarray jbyteArray;
typedef jarray jintArray;
typedef jarray jlongArray;
#define JNI_ABORT 2
#define JNIEXPORT __attribute__((visibility("default")))
#define JNICALL

struct JNINativeInterface_;
typedef const struct JNINativeInterface_* JNIEnv;
struct JNINativeInterface_ {
  jclass (*FindClass)(JNIEnv*, const char*);
  jint (*ThrowNew)(JNIEnv*, jclass, const char*);
  jboolean (*ExceptionCheck)(JNIEnv*);
  void (*DeleteLocalRef)(JNIEnv*, jobject);
  jsize (*GetArrayLength)(JNIEnv*, jarray);
  jobject (*GetObjectArrayElement)(JNIEnv*, jobjectArray, jsize);
  jlong* (*GetLongArrayElements)(JNIEnv*, jlongArray, jboolean*);
  void (*ReleaseLongArrayElements)(JNIEnv*, jlongArray, jlong*, jint);
  jint* (*GetIntArrayElements)(JNIEnv*, jintArray, jboolean*);
  void (*ReleaseIntArrayElements)(JNIEnv*, jintArray, jint*, jint);
  void (*GetByteArrayRegion)(JNIEnv*, jbyteArray, jsize, jsize, jbyte*);
  void (*SetByteArrayRegion)(JNIEnv*, jbyteArray, jsize, jsize, const jbyte*);
  void (*SetLongArrayRegion)(JNIEnv*, jlongArray, jsize, jsize, const jlong*);
};
#endif
